"""TEST INFRASTRUCTURE ONLY -- CPU (PyTorch fp32) restatement of the MelGAN generators and PQMF synthesis over a
reference-format state dict, the checker for tts_b200.melgan:

  generator(sd, c, ...)   MelganGenerator.forward (TTS/vocoder/models/melgan_generator.py:9-74, ResidualStack
                          TTS/vocoder/layers/melgan.py:6-36): the same layers for all three generators
  inference(sd, c, ...)   replicate pad of 2 frames, the layers and, with ``pqmf=True``, PQMF synthesis
  pqmf_synthesis(G, x)    PQMF.synthesis (TTS/vocoder/layers/pqmf.py:50-53)

Every conv with kernel > 1 reflect-pads (F.pad mode "reflect"); the transposed convs and 1x1 convs do not pad, and the
PQMF filter zero-pads.  Pinned ``torch.equal`` to the unmodified reference by tests/test_melgan_oracle_cpu.py."""
import torch
import torch.nn.functional as F

from vits_oracle import conv_weight, sub

SLOPE = 0.2


def layer_indices(n_up):
    """Indices in ``layers`` of conv_pre, each stage's (upsampler, residual stack), and conv_post."""
    return 1, [(3 + 3 * s, 4 + 3 * s) for s in range(n_up)], 3 * n_up + 4


def _conv(sd, name, x, *, dilation=1, reflect=0):
    if reflect:
        x = F.pad(x, (reflect, reflect), mode="reflect")
    return F.conv1d(x, conv_weight(sd, name), sd[name + ".bias"], dilation=dilation)


def residual_stack(sd, x, *, num_res_blocks, res_kernel):
    for m in range(num_res_blocks):
        d = res_kernel ** m
        h = _conv(sd, f"blocks.{m}.2", F.leaky_relu(x, SLOPE), dilation=d, reflect=(res_kernel - 1) // 2 * d)
        h = _conv(sd, f"blocks.{m}.4", F.leaky_relu(h, SLOPE))
        x = _conv(sd, f"shortcuts.{m}", x) + h
    return x


def generator(sd, c, *, upsample_factors, num_res_blocks, proj_kernel=7, res_kernel=3):
    """``self.layers(c)``: [B, in, T] -> [B, out, T * prod(upsample_factors)]."""
    sd = sub(sd, "layers")
    pre, stages, post = layer_indices(len(upsample_factors))
    pad = (proj_kernel - 1) // 2
    x = _conv(sd, str(pre), c, reflect=pad)
    for u, (iu, ir) in zip(upsample_factors, stages):
        w = conv_weight(sd, str(iu))
        x = F.conv_transpose1d(F.leaky_relu(x, SLOPE), w, sd[f"{iu}.bias"], stride=u, padding=u // 2 + u % 2,
                               output_padding=u % 2)
        x = residual_stack(sub(sd, str(ir)), x, num_res_blocks=num_res_blocks, res_kernel=res_kernel)
    return torch.tanh(_conv(sd, str(post), F.leaky_relu(x, SLOPE), reflect=pad))


def pqmf_synthesis(G, x):
    """[B, N, Tb] -> [B, 1, N * Tb]: zero-stuff by N (scaled by N), then the synthesis filter G [1, N, taps + 1] with
    taps / 2 zeros each side."""
    n = x.shape[1]
    taps = G.shape[-1] - 1
    up = torch.zeros(x.shape[0], n, x.shape[2] * n, dtype=x.dtype, device=x.device)
    up[:, :, ::n] = x * n
    return F.conv1d(up, G, padding=taps // 2)


def inference(sd, c, *, pqmf=False, padding=2, **kw):
    y = generator(sd, F.pad(c, (padding, padding), mode="replicate"), **kw)
    return pqmf_synthesis(sd["pqmf_layer.G"], y) if pqmf else y
