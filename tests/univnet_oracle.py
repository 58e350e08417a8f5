"""TEST INFRASTRUCTURE ONLY -- CPU (PyTorch) restatement of UnivnetGenerator.forward over a reference-format state dict,
the checker for tts_b200.univnet:

  kernel_predictor(sd, p, c, ...)     KernelPredictor (TTS/vocoder/layers/lvc_block.py): input_conv + LeakyReLU(0.1),
                                      c + residual_conv(c), then kernel_conv / bias_conv -> kernels [B, L, Cin, Cout, K, T],
                                      biases [B, L, Cout, T]
  lvc(y, kernels, bias, hop)          the location-variable convolution: output sample s of frame f = s // hop is
                                      sum_ci sum_k kernels[ci, co, k, f] y[ci, s + k - 1] + bias[co, f], y zero-padded
                                      only at the row ends
  generator(sd, c, noise, ...)        UnivnetGenerator.forward on given noise [B, in_channels, T]

Device- and dtype-agnostic (float64 on the GPU for the kernel tests, fp32 on the CPU for the parity tests).  Pinned
``torch.equal`` to the unmodified reference by tests/test_univnet_oracle_cpu.py."""
import torch
import torch.nn.functional as F

from vits_oracle import conv_weight

RESIDUAL_CONVS = (1, 3, 6, 8, 11, 13)


def kernel_predictor(sd, p, c, *, layers, hidden, kernel_size=3):
    k = sd[p + "kernel_conv.bias"].numel()
    kp = conv_weight(sd, p + "kernel_conv").shape[-1]
    pad = (kp - 1) // 2
    h = F.leaky_relu(F.conv1d(c, conv_weight(sd, p + "input_conv.0"), sd[p + "input_conv.0.bias"], padding=2), 0.1)
    r = h
    for i in RESIDUAL_CONVS:
        q = f"{p}residual_conv.{i}"
        r = F.leaky_relu(F.conv1d(r, conv_weight(sd, q), sd[q + ".bias"], padding=pad), 0.1)
    h = h + r
    kern = F.conv1d(h, conv_weight(sd, p + "kernel_conv"), sd[p + "kernel_conv.bias"], padding=pad)
    bias = F.conv1d(h, conv_weight(sd, p + "bias_conv"), sd[p + "bias_conv.bias"], padding=pad)
    b, _, t = c.shape
    assert k == layers * hidden * 2 * hidden * kernel_size
    return kern.view(b, layers, hidden, 2 * hidden, kernel_size, t), bias.view(b, layers, 2 * hidden, t)


def lvc(y, kernels, bias, hop):
    """y [B, Cin, T * hop], kernels [B, Cin, Cout, K, T], bias [B, Cout, T] -> [B, Cout, T * hop] (dilation 1)."""
    b, cin, n = y.shape
    t, ksz = kernels.shape[-1], kernels.shape[3]
    pad = (ksz - 1) // 2
    yp = F.pad(y, (pad, pad))
    win = torch.stack([yp[:, :, k:k + n] for k in range(ksz)], dim=-1).view(b, cin, t, hop, ksz)   # y[s + k - pad]
    out = torch.einsum("bifhk,biokf->bofh", win, kernels)
    return (out + bias.unsqueeze(-1)).reshape(b, -1, n)


def lvc_layer(sd, p, i, x, kernels, bias, hop):
    """One LVC layer of block prefix p: x + sigmoid(o[:C]) tanh(o[C:]), o = LVC(lrelu(conv_i(lrelu(x, 0.2)), 0.2))."""
    d = 3 ** i
    q = f"{p}convs.{i}"
    w = conv_weight(sd, q)
    y = F.leaky_relu(F.conv1d(F.leaky_relu(x, 0.2), w, sd[q + ".bias"], padding=d * (w.shape[-1] - 1) // 2, dilation=d),
                     0.2)
    o = lvc(y, kernels, bias, hop)
    ch = x.shape[1]
    return x + torch.sigmoid(o[:, :ch]) * torch.tanh(o[:, ch:])


def generator(sd, c, noise, *, upsample_factors=(8, 8, 4), layers=4):
    """c [B, cond, T], noise [B, in_channels, T] -> [B, out_channels, T * prod(upsample_factors)]."""
    x = F.conv1d(noise, conv_weight(sd, "first_conv"), sd["first_conv.bias"], padding=3)
    hidden = x.shape[1]
    hop = 1
    for n, u in enumerate(upsample_factors):
        hop *= u
        p = f"lvc_blocks.{n}."
        kernels, bias = kernel_predictor(sd, p + "kernel_predictor.", c, layers=layers, hidden=hidden)
        x = F.conv_transpose1d(F.leaky_relu(x, 0.2), sd[p + "upsample.weight"], sd[p + "upsample.bias"], stride=u,
                               padding=u // 2 + u % 2, output_padding=u % 2)
        for i in range(layers):
            x = lvc_layer(sd, p, i, x, kernels[:, i], bias[:, i], hop)
    x = F.conv1d(F.leaky_relu(x, 0.1), conv_weight(sd, "last_conv_layers.0"), sd["last_conv_layers.0.bias"], padding=3)
    return torch.tanh(x)
