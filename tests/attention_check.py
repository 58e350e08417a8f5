"""Float64 restatements of the transformer layers' attention and add + LayerNorm kernels, and the bounds their outputs
are held to (``test_attention_edges_gpu.py``).

- ``rel_attention`` is the FP32-FMA attention core (``b200tts_debug_attention``): the closed form of
  ``oracle/vits_oracle.py:rel_attention`` without the q / k / v / o convs, over a fused [B, 3C, T] q|k|v tensor.
- ``attention_tc3`` is the tensor-core attention core (``b200tts_attention_tc3``): a per-row softmax over the first
  lens[b] keys, zero output from lens[b] to the pitch.
- ``add_layernorm`` is both add + LayerNorm kernels (``b200tts_debug_add_layernorm`` kinds 0 and 1).

Each takes a ``dtype``: float64 is the reference, float32 is torch's own fp32 result on the same inputs, the yardstick
of the bound.  ``test_attention_checker_cpu.py`` pins these restatements to the oracle and to torch, and shows that
``failures`` rejects a set of near-miss mistakes.

Test infrastructure only; it works on whatever device its inputs live on.
"""
import math

import torch

# The bound, stated before any kernel was measured against it.  Per slice (a batch row of an attention output, one
# column of a LayerNorm output), the RMS error of the kernel vs float64 must be
#   <= FP32_FACTOR x the RMS error of torch's fp32 computation of the same thing (the kernel is "as accurate as fp32";
#      FP32_FACTOR = 2 leaves room for a different summation order, not for a lost term or a wrong constant), or
#   <= REL_FLOOR x the slice's RMS (for slices torch happens to get almost exact: a few fp32 ulps of the result).
FP32_FACTOR = 2.0
REL_FLOOR = 1e-5
# LayerNorm only: a column whose mean is far from zero (|mean| / std = kappa) loses accuracy in any fp32 two-pass
# LayerNorm.  The mean is a sum of C values of size ~|mean|, summed by each of 8 channel groups and then across them
# (at most C / 8 + 8 roundings, each <= 2^-24 of the running sum), and x + y (+ y) adds up to two roundings of size
# 2^-24 |mean| per element.  An error d in the mean moves every normalized value by d / std.  Hence the per-element
# bound (LN_TERMS(C) x 2^-24 x kappa x max|gamma|).  A one-pass variance (E[v^2] - mean^2) instead loses the variance
# itself once kappa^2 2^-24 is near 1 (kappa = 1e5 in the sweep's offset column): its error is O(1) or NaN.
LN_GROUPS = 8


def ln_terms(c):
    return math.ceil(c / LN_GROUPS) + LN_GROUPS + 2


def _split(qkv, heads, dtype):
    b, c3, t = qkv.shape
    c = c3 // 3
    d = c // heads
    q, k, v = (qkv[:, s * c:(s + 1) * c].to(dtype).reshape(b, heads, d, t).transpose(2, 3) for s in range(3))
    return q, k, v, d   # [b, h, t, d]


def rel_attention(qkv, mask, heads, window=-1, rel_k=None, rel_v=None, dtype=torch.float64):
    """out [B, C, T] of the FMA attention core: s_ij = (q_i.k_j + [|j-i| <= w] q_i.rel_k[j-i+w]) / sqrt(d), then
    masked_fill(mask_i mask_j == 0, -1e4) over the whole padded length, softmax over all T keys (a padded query row is
    uniform), out_i = sum_j p_ij v_j + sum_{|j-i| <= w} p_ij rel_v[j-i+w].  rel_k / rel_v [2w+1, d]; window -1: none."""
    q, k, v, d = _split(qkv, heads, dtype)
    b, h, t, _ = q.shape
    scores = torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(d)
    if window >= 0:
        idx = torch.arange(t, device=qkv.device)
        off = idx[None, :] - idx[:, None] + window                # j - i + w
        band = (off >= 0) & (off <= 2 * window)
        offc = off.clamp(0, 2 * window).expand(b, h, t, t)
        rel = torch.matmul(q, rel_k.to(dtype).t()) / math.sqrt(d)  # [b, h, t, 2w+1]
        scores = scores + torch.where(band, torch.gather(rel, 3, offc), torch.zeros((), dtype=dtype, device=q.device))
    m = mask.to(dtype)
    keep = (m[:, None, :, None] * m[:, None, None, :]) != 0
    scores = scores.masked_fill(~keep, -1e4)
    p = torch.softmax(scores, -1)
    out = torch.matmul(p, v)
    if window >= 0:
        # p on the band, gathered per relative offset r: pw[..., i, r] = p[..., i, i + r - w] (0 off the ends)
        r = torch.arange(2 * window + 1, device=qkv.device)
        j = idx[:, None] + r[None, :] - window                    # [t, 2w+1]
        inside = (j >= 0) & (j < t)
        pw = torch.gather(p, 3, j.clamp(0, t - 1).expand(b, h, t, 2 * window + 1))
        pw = torch.where(inside, pw, torch.zeros((), dtype=dtype, device=q.device))
        out = out + torch.matmul(pw, rel_v.to(dtype))
    return out.transpose(2, 3).reshape(b, h * d, t)


def attention_tc3(qkv, lens, heads, pitch=None, dtype=torch.float64):
    """out [B, C, pitch] of the tensor-core attention core: per row b, softmax((q * d^-1/2) k^T) v over its first
    lens[b] frames (q scaled first, as torch's MultiheadAttention), zero from lens[b] to the pitch.  qkv [B, 3C, pitch];
    its columns at or past lens[b] are never used."""
    b, c3, t = qkv.shape
    pitch = t if pitch is None else pitch
    c = c3 // 3
    d = c // heads
    out = torch.zeros(b, c, pitch, dtype=dtype, device=qkv.device)
    for i in range(b):
        n = min(int(lens[i]), pitch)
        if n <= 0:
            continue
        q, k, v = (qkv[i, s * c:(s + 1) * c, :n].to(dtype).reshape(heads, d, n) for s in range(3))
        p = torch.softmax(torch.einsum("hci,hcj->hij", q * math.sqrt(1.0 / d), k), -1)
        out[i, :, :n] = torch.einsum("hij,hcj->hci", p, v).reshape(c, n)
    return out


def add_layernorm(x, y, gamma, beta, mask=None, *, eps, twice=False, select=False, dtype=torch.float64):
    """out [B, C, T]: v = x + y (+ y again when twice; y None: v = x), LayerNorm over the C channels with the biased
    variance, (v - mean) / sqrt(var + eps) * gamma + beta.  Kind 0 multiplies by mask[b, t] (None: 1); kind 1
    (select=True) yields an exact 0 where mask[b, t] == 0, whatever x and y hold there."""
    v = x.to(dtype)
    if y is not None:
        v = v + y.to(dtype)
        if twice:
            v = v + y.to(dtype)
    mean = v.mean(1, keepdim=True)
    var = (v - mean).pow(2).mean(1, keepdim=True)
    out = (v - mean) / torch.sqrt(var + eps) * gamma.to(dtype)[None, :, None] + beta.to(dtype)[None, :, None]
    if mask is None:
        return out
    m = mask.to(dtype)[:, None, :]
    if select:
        return torch.where(m != 0, out, torch.zeros((), dtype=dtype, device=out.device))
    return out * m


def _rms(t, dims):
    return t.pow(2).mean(dims).sqrt()


def failures(got, want, f32, dims, extra=None):
    """Indices of the slices (the dimensions not in ``dims``) whose error breaks the bound above; ``extra``: an added
    per-slice allowance (the LayerNorm offset term).  NaN anywhere in a slice breaks it."""
    g, w, f = got.double(), want.double(), f32.double()
    err, err32, scale = _rms(g - w, dims), _rms(f - w, dims), _rms(w, dims)
    bound = torch.maximum(FP32_FACTOR * err32, REL_FLOOR * scale)
    if extra is not None:
        bound = torch.maximum(bound, extra)
    bad = ~(err <= bound)   # NaN compares false
    return [tuple(int(i) for i in ix) for ix in bad.nonzero()], err, bound


def attention_failures(got, want, f32, cols=None):
    """Batch rows of [B, C, T] attention outputs over their first cols[b] columns (all columns when None)."""
    out = []
    for b in range(got.shape[0]):
        n = got.shape[2] if cols is None else int(cols[b])
        if n > 0 and failures(got[b:b + 1, :, :n], want[b:b + 1, :, :n], f32[b:b + 1, :, :n], (1, 2))[0]:
            out.append(b)
    return out


def ln_offset_allowance(x, y, gamma, twice=False):
    """Per column: the offset term of the LayerNorm bound, LN_TERMS(C) * 2^-24 * |mean| / std * max|gamma| (0 for a
    constant column, and for one that is not finite: a masked column of kind 1 must come out exactly 0)."""
    v = x.double() + (0 if y is None else y.double() * (2 if twice else 1))
    mean = v.mean(1)
    std = (v - mean[:, None]).pow(2).mean(1).sqrt()
    kappa = torch.where(std > 0, mean.abs() / std.clamp_min(1e-300), torch.zeros_like(std))
    return torch.nan_to_num(ln_terms(x.shape[1]) * 2.0 ** -24 * kappa * float(gamma.abs().max()), nan=0.0, posinf=0.0)


def layernorm_failures(got, want, f32, x, y, gamma, twice=False):
    """(batch, column) pairs of [B, C, T] LayerNorm outputs that break the bound (per column over its C channels)."""
    return failures(got, want, f32, (1,), ln_offset_allowance(x, y, gamma, twice))[0]
