"""TEST INFRASTRUCTURE ONLY -- CPU (PyTorch fp32) restatement of the WaveGrad vocoder over a reference-format state dict,
the checker for tts_b200.wavegrad (runs on any device: the benchmark also runs it eagerly on the GPU):

  forward(sd, y, spec, noise_scale, args)   Wavegrad.forward (TTS/vocoder/models/wavegrad.py:106-120; DBlock, FiLM,
                                            UBlock, PositionalEncoding: TTS/vocoder/layers/wavegrad.py:19-154)
  schedule(beta)                            Wavegrad.compute_noise_level (wavegrad.py:160-176)
  inference(sd, spec, sched, args, ...)     Wavegrad.inference (wavegrad.py:126-145) with the reference's draw order, or
                                            supplied noise (step_noise[n - 1] is the z of step n)

``args``: a WavegradArgs-like object (attribute access).  Weight-normed keys (parametrizations or legacy weight_g / _v)
are folded as torch folds them.  Pinned ``torch.equal`` to the unmodified reference by tests/test_wavegrad_oracle_cpu.py."""
import numpy as np
import torch
import torch.nn.functional as F

from vits_oracle import conv_weight, sub

SLOPE = 0.2


def _conv(sd, name, x, dilation=1, padding=0):
    return F.conv1d(x, conv_weight(sd, name), sd[name + ".bias"], dilation=dilation, padding=padding)


def pe_table(n_channels, length):
    """PositionalEncoding.init_pe_matrix (CPU float32)."""
    pe = torch.zeros(length, n_channels)
    position = torch.arange(0, length, dtype=torch.float).unsqueeze(1)
    div_term = torch.pow(10000, torch.arange(0, n_channels, 2).float() / n_channels)
    pe[:, 0::2] = torch.sin(position / div_term)
    pe[:, 1::2] = torch.cos(position / div_term)
    return pe.transpose(0, 1)


def film(sd, x, noise_scale):
    o = F.leaky_relu(_conv(sd, "input_conv", x, padding=1), SLOPE)
    pe = pe_table(o.shape[1], o.shape[2]).to(o)
    o = o + noise_scale[..., None, None] + pe[:, : o.size(2)].repeat(o.shape[0], 1, 1) / 5000
    return torch.chunk(_conv(sd, "output_conv", o, padding=1), 2, dim=1)


def dblock(sd, x, factor):
    size = x.shape[-1] // factor
    res = F.interpolate(_conv(sd, "res_block", x), size=size)
    o = F.interpolate(x, size=size)
    for i, d in enumerate((1, 2, 4)):
        o = _conv(sd, f"main_block.{i}", F.leaky_relu(o, SLOPE), dilation=d, padding=d)
    return o + res


def ublock(sd, x, shift, scale, factor, dilation):
    x_inter = F.interpolate(x, size=x.shape[-1] * factor)
    res = _conv(sd, "res_block", x_inter)
    o = _conv(sd, "main_block.0", F.leaky_relu(x_inter, SLOPE), dilation[0], dilation[0])
    o = shift + scale * o
    res2 = res + _conv(sd, "main_block.1", F.leaky_relu(o, SLOPE), dilation[1], dilation[1])
    o = shift + scale * res2
    o = _conv(sd, "out_block.0", F.leaky_relu(o, SLOPE), dilation[2], dilation[2])
    o = shift + scale * o
    return _conv(sd, "out_block.1", F.leaky_relu(o, SLOPE), dilation[3], dilation[3]) + res2


def forward(sd, y, spec, noise_scale, args, cond=None):
    """``cond``: x_conv(spec), when the caller has it already (the refinement loop computes it once)."""
    pairs = []
    x = _conv(sd, "y_conv", y, padding=2)
    pairs.append(film(sub(sd, "film.0"), x, noise_scale))
    for i, df in enumerate(list(reversed(args.upsample_factors))[: len(args.dblock_out_channels)]):
        x = dblock(sub(sd, f"dblocks.{i}"), x, df)
        pairs.append(film(sub(sd, f"film.{i + 1}"), x, noise_scale))
    x = _conv(sd, "x_conv", spec, padding=1) if cond is None else cond
    for j, (shift, scale) in enumerate(reversed(pairs)):
        x = ublock(sub(sd, f"ublocks.{j}"), x, shift, scale, args.upsample_factors[j], args.upsample_dilations[j])
    return _conv(sd, "out_conv", x, padding=1)


def schedule(beta):
    """compute_noise_level: {beta, alpha, alpha_hat, noise_level, c1, c2, sigma} as float32 CPU tensors."""
    alpha = 1 - beta
    alpha_hat = np.cumprod(alpha)
    noise_level = alpha_hat**0.5
    s = {k: torch.tensor(v.astype(np.float32)) for k, v in
         (("beta", beta), ("alpha", alpha), ("alpha_hat", alpha_hat), ("noise_level", noise_level))}
    s["c1"] = 1 / s["alpha"] ** 0.5
    s["c2"] = (1 - s["alpha"]) / (1 - s["alpha_hat"]) ** 0.5
    s["sigma"] = ((1.0 - s["alpha_hat"][:-1]) / (1.0 - s["alpha_hat"][1:]) * s["beta"][1:]) ** 0.5
    return s


def inference(sd, spec, sched, args, init_noise=None, step_noise=None):
    """The refinement loop.  Without ``init_noise`` the start is ``torch.randn`` on the CPU generator, without
    ``step_noise`` every step n > 0 draws ``torch.randn_like(y)`` -- the reference's order.  x_conv runs once (its input
    is the same at every step, so this is the same arithmetic)."""
    hop = int(np.prod(args.upsample_factors))
    y = torch.randn(spec.shape[0], 1, hop * spec.shape[-1]) if init_noise is None else init_noise
    y = y.type_as(spec)
    level = sched["noise_level"].to(spec)
    cond = _conv(sd, "x_conv", spec, padding=1)
    for n in range(len(sched["alpha"]) - 1, -1, -1):
        y = sched["c1"][n] * (y - sched["c2"][n] * forward(sd, y, spec, level[n].repeat(spec.shape[0]), args, cond))
        if n > 0:
            z = torch.randn_like(y) if step_noise is None else step_noise[n - 1].to(y)
            y += sched["sigma"][n - 1] * z
        y.clamp_(-1.0, 1.0)
    return y
