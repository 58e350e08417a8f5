"""TEST INFRASTRUCTURE ONLY -- CPU (PyTorch) restatement of ParallelWaveganGenerator.forward over a reference-format state
dict, the checker for tts_b200.pwgan:

  upsample(sd, c, factors)            ConvUpsample.forward (TTS/vocoder/layers/upsample.py): conv_in, then per factor
                                      F.interpolate nearest (1, u) and the (1, 2u + 1) conv with zero padding u
  generator(sd, c, noise, ...)        ParallelWaveganGenerator.forward (TTS/vocoder/models/parallel_wavegan_generator.py:
                                      93-121; ResidualBlock TTS/vocoder/layers/parallel_wavegan.py:49-82) on given noise
  inference(sd, c, noise, ...)        replicate pad of ``padding`` frames, then ``generator``

Device- and dtype-agnostic (float64 on the GPU for the kernel tests, fp32 on the CPU for the parity tests).  Pinned
``torch.equal`` to the unmodified reference by tests/test_pwgan_oracle_cpu.py."""
import math

import torch
import torch.nn.functional as F

from vits_oracle import conv_weight


def stages(sd, c, upsample_factors):
    """The stage chain of UpsampleNetwork on [B, C, T] -> [B, C, T * prod(factors)]."""
    c = c.unsqueeze(1)
    for i, u in enumerate(upsample_factors):
        c = F.interpolate(c, scale_factor=(1, u), mode="nearest")
        c = F.conv2d(c, conv_weight(sd, f"upsample_net.upsample.up_layers.{2 * i + 1}"), padding=(0, u))
    return c.squeeze(1)


def upsample(sd, c, upsample_factors):
    return stages(sd, F.conv1d(c, conv_weight(sd, "upsample_net.conv_in")), upsample_factors)


def generator(sd, c, noise, *, upsample_factors=(4, 4, 4, 4), num_res_blocks=30, stacks=3):
    """c [B, 80, T], noise [B, 1, T * prod(upsample_factors)] -> [B, 1, T * prod(upsample_factors)]."""
    x = F.conv1d(noise, conv_weight(sd, "first_conv"), sd["first_conv.bias"])
    c = upsample(sd, c, upsample_factors)
    per_stack = num_res_blocks // stacks
    skips = 0
    for layer in range(num_res_blocks):
        p = f"conv_layers.{layer}."
        d = 2 ** (layer % per_stack)
        residual = x
        h = F.conv1d(x, conv_weight(sd, p + "conv"), sd[p + "conv.bias"], padding=d, dilation=d)
        xa, xb = h.split(h.size(1) // 2, dim=1)
        a = F.conv1d(c, conv_weight(sd, p + "conv1x1_aux"))
        ca, cb = a.split(a.size(1) // 2, dim=1)
        z = torch.tanh(xa + ca) * torch.sigmoid(xb + cb)
        s = F.conv1d(z, conv_weight(sd, p + "conv1x1_skip"), sd[p + "conv1x1_skip.bias"])
        x = (F.conv1d(z, conv_weight(sd, p + "conv1x1_out"), sd[p + "conv1x1_out.bias"]) + residual) * (0.5 ** 2)
        skips += s
    skips *= math.sqrt(1.0 / num_res_blocks)
    x = F.relu(skips)
    x = F.conv1d(x, conv_weight(sd, "last_conv_layers.1"), sd["last_conv_layers.1.bias"])
    x = F.relu(x)
    return F.conv1d(x, conv_weight(sd, "last_conv_layers.3"), sd["last_conv_layers.3.bias"])


def inference(sd, c, noise, *, padding=2, **kw):
    return generator(sd, F.pad(c, (padding, padding), mode="replicate"), noise, **kw)
