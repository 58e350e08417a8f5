"""The transformer layers' attention and add + LayerNorm kernels against float64 (attention_check.py), one launch at a
time, at the edges of their tiles and dispatch rules.

- ``attention_tc3_kernel`` (ForwardTTS decoder, dispatch id ``attn_tc3``): head widths around its 64-channel S chunks
  and its 4-warp channel n-tile groups (d / 8 % 4 != 0), T around FA_BQ = 32 / FA_BK = 64 up to the decoder's 5000
  frames, rows of length 0 / 1 / 63 / 64 / 65 / T, pitches T, ceil4(T) (the decoder) and T + 100, NaN in q|k|v past
  each row's end, and three score ranges: +-80, the row maximum in the last key tile (the online rescale on every
  tile) and all scores equal.
- ``rel_attention_kernel<256>`` / ``<384>`` (VITS / Glow-TTS / ForwardTTS text encoders and the decoder fallback,
  ``b200tts_debug_attention``, dispatch id ``attn_fma``): d across both instantiations and partial lanes, every
  relative window up to 15, T around ATT_Q = 8 / ATT_KT = 32 and the largest T its shared memory takes, ragged masks
  with an all-zero row, and +-1e6 in every padded column (valid outputs must not move: bit-identical to zeros there).
- ``add_layernorm_kernel`` (kind 0) and ``fft_add_norm_kernel`` (kind 1, ``b200tts_debug_add_layernorm``): C around
  the 8 channel groups, T around the 32-column blocks, y / mask present and absent, eps 1e-4 / 1e-5, in place as the
  layers run them, a column with mean 1e3 and spread 1e-2, and NaN in the masked columns of kind 1.

Outputs are NaN-prefilled, so a column no thread writes shows up.  The bound is attention_check's (stated there before
any measurement).  Exact properties: a relaunch is bit-identical, a ragged row equals the single-row call on its valid
columns, and the columns the contracts zero are exactly zero.  Rejections are host-side: an error and no launch.
"""
import math

import pytest
import torch

import attention_check as AC
from tts_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NAN = float("nan")

# shared-memory budget of the FMA attention kernel (text_encoder.cu: launch_attention), in floats
FMA_SMEM_FLOATS = 200 * 1024 // 4


def fma_max_t(d, window):
    """largest T whose shared memory fits: 8 d + 8 Tp + 33 (d + 1) + 2 nrel d floats, Tp = ceil32(T)"""
    nrel = 0 if window < 0 else 2 * window + 1
    return (FMA_SMEM_FLOATS - 8 * d - 33 * (d + 1) - 2 * nrel * d) // 8 // 32 * 32


def ceil4(t):
    return (t + 3) // 4 * 4


def _f32_no_tf32(fn):
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def _tf32(fn):
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


# ------------------------------------------------------------------------------------------------ launchers
def run_tc3(qkv, lens, heads, t, out=None):
    """b200tts_attention_tc3 over qkv [B, 3C, pitch] into a NaN-prefilled out [B, C, pitch]"""
    b, c3, pitch = qkv.shape
    c = c3 // 3
    out = torch.full((b, c, pitch), NAN, device=DEV) if out is None else out
    ln = torch.as_tensor(lens, dtype=torch.int32, device=DEV)
    rc = _lib.lib().b200tts_attention_tc3(_lib.ptr(qkv), _lib.ptr(ln), b, c, heads, t, pitch, _lib.ptr(out),
                                          _lib.stream_ptr(DEV))
    _lib.check(rc, "attention_tc3")
    return out


def run_fma(qkv, mask, heads, window, ek=None, ev=None):
    b, c3, t = qkv.shape
    c = c3 // 3
    out = torch.full((b, c, t), NAN, device=DEV)
    rc = _lib.lib().b200tts_debug_attention(_lib.ptr(qkv), _lib.ptr(mask), _lib.ptr(ek), _lib.ptr(ev), _lib.ptr(out), b,
                                            c, t, heads, window, _lib.stream_ptr(DEV))
    _lib.check(rc, "debug_attention")
    return out


def run_ln(kind, x, y, gamma, beta, mask, eps, twice=False, out=None):
    """in place (out = x) unless out is given"""
    b, c, t = x.shape
    out = x if out is None else out
    rc = _lib.lib().b200tts_debug_add_layernorm(kind, _lib.ptr(x), _lib.ptr(y), int(twice), _lib.ptr(gamma),
                                                _lib.ptr(beta), _lib.ptr(mask), _lib.ptr(out), b, c, t, eps,
                                                _lib.stream_ptr(DEV))
    _lib.check(rc, "debug_add_layernorm")
    return out


# ------------------------------------------------------------------------------------------------ attention_tc3
TC3_D = [8, 16, 56, 64, 72, 120, 128, 136, 192, 200, 256, 264, 328, 376, 384]
TC3_T = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1000, 5000]
TC3_LENS = [0, 1, 63, 64, 65]
SCORES = ["normal", "wide", "last_tile_max", "flat"]


def tc3_cases():
    """every (d, T) pair; heads, batch, the other rows' lengths, the pitch and the score range rotate over the pairs
    so that each value of each meets many of the others"""
    cases = []
    for i, d in enumerate(TC3_D):
        for j, t in enumerate(TC3_T):
            k = i + j
            heads = 1 + k % 4
            b = 1 + (i + 2 * j) % 3
            pitch = [t, ceil4(t), t + 100][k % 3]
            lens = [t] + [min(TC3_LENS[(k + r) % 5], t) for r in range(b - 1)]
            cases.append(pytest.param(d, heads, t, pitch, lens, SCORES[(i + 3 * j) % 4],
                                      id=f"d{d}_h{heads}_t{t}_p{pitch}_l{'-'.join(map(str, lens))}_{SCORES[(i + 3 * j) % 4]}"))
    return cases


def tc3_inputs(d, heads, pitch, lens, scores, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = d * heads
    qkv = torch.randn(len(lens), 3 * c, pitch, generator=g, device=DEV)
    if scores == "wide":        # q . k d^-1/2 ~ N(0, 20^2): the scores span about +-80
        qkv[:, :c] *= 20.0
    elif scores == "flat":      # q = 0: every score 0, the output is the mean of v
        qkv[:, :c] = 0.0
    elif scores == "last_tile_max":
        # q ~ 1, k_j ~ (8 j / n) d^-1/2: scores ~ 8 j / n rise over the keys, every key tile holds a new row maximum
        qkv[:, :c] = 1.0 + 0.1 * qkv[:, :c]
        for i, n in enumerate(lens):
            ramp = 8.0 * torch.arange(pitch, device=DEV) / max(n, 1) / math.sqrt(d)
            qkv[i, c:2 * c] = ramp[None, :] + 0.1 * qkv[i, c:2 * c] / math.sqrt(d)
    for i, n in enumerate(lens):   # stale scratch past a row's end is never read
        qkv[i, :, n:] = NAN
    return qkv


@pytest.mark.parametrize("d,heads,t,pitch,lens,scores", tc3_cases())
def test_attention_tc3_against_float64(d, heads, t, pitch, lens, scores):
    qkv = tc3_inputs(d, heads, pitch, lens, scores, seed=d * 7919 + t * 31 + pitch)
    with _lib.dispatch_log() as log:
        got = run_tc3(qkv, lens, heads, t)
    assert log.names == ["attn_tc3"]
    clean = torch.nan_to_num(qkv)
    want = AC.attention_tc3(clean, lens, heads)
    f32 = _f32_no_tf32(lambda: AC.attention_tc3(clean, lens, heads, dtype=torch.float32))
    for i, n in enumerate(lens):   # zero from the row's end up to the pitch, the columns past ceil32(T) included
        tail = got[i, :, n:]
        assert torch.equal(tail, torch.zeros_like(tail)), (i, n, int(tail.isnan().sum()))
    assert not AC.attention_failures(got, want, f32, cols=lens)
    assert torch.equal(run_tc3(qkv, lens, heads, t), got)   # a relaunch is bit-identical
    for i, n in enumerate(lens[1:], 1):                       # a ragged row equals its single-row call
        if n > 0:
            one = run_tc3(qkv[i:i + 1, :, :n].contiguous(), [n], heads, n)
            assert torch.equal(one[0], got[i, :, :n]), i
    if t >= 1000:   # the bound discriminates: single-pass TF32 products of the same attention break it
        tf32 = _tf32(lambda: AC.attention_tc3(clean, lens, heads, dtype=torch.float32))
        assert AC.attention_failures(tf32[:1], want[:1], f32[:1], cols=lens[:1])


def test_attention_tc3_zeroes_the_whole_pitch_of_empty_rows():
    """T = 0 under a pitch of 40: every output column is a padded column and must come out 0"""
    qkv = torch.full((2, 3 * 64, 40), NAN, device=DEV)
    got = run_tc3(qkv, [0, 0], 2, 0)
    assert torch.equal(got, torch.zeros_like(got))


# ------------------------------------------------------------------------------------------------ FMA attention
FMA_D = [1, 2, 31, 32, 33, 96, 255, 256, 257, 300, 384]
FMA_T = [1, 2, 4, 5, 7, 8, 9, 31, 32, 33, 64, 65]
WINDOWS = [-1, 0, 1, 4, 15]


def fma_cases():
    cases = []
    for i, d in enumerate(FMA_D):
        for j, t in enumerate(FMA_T):
            k = i + j
            window = WINDOWS[k % 5]
            heads = 1 + (i + 2 * j) % 3
            b = 1 + k % 3
            lens = [t, 0, t // 2 + 1][:b] if k % 2 else [t, max(t - 1, 1), 1][:b]
            cases.append(pytest.param(d, heads, window, t, lens, id=f"d{d}_h{heads}_w{window}_t{t}_l{'-'.join(map(str, lens))}"))
    # the largest T the kernel's shared memory takes: VITS (d 96, window 4) and ForwardTTS's text encoder (d 384)
    for d, heads, window in ((96, 2, 4), (384, 1, -1)):
        t = fma_max_t(d, window)
        cases.append(pytest.param(d, heads, window, t, [t, t - 333], id=f"d{d}_h{heads}_w{window}_tmax{t}"))
    return cases


def fma_inputs(d, heads, window, t, lens, seed, pad_value):
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = d * heads
    qkv = torch.randn(len(lens), 3 * c, t, generator=g, device=DEV)
    mask = (torch.arange(t, device=DEV)[None, :] < torch.tensor(lens, device=DEV)[:, None]).float()
    ek = ev = None
    if window >= 0:
        ek = torch.randn(2 * window + 1, d, generator=g, device=DEV)
        ev = torch.randn(2 * window + 1, d, generator=g, device=DEV)
    garbage = torch.where(torch.rand(qkv.shape, generator=g, device=DEV) < 0.5, -1.0, 1.0) * 1e6
    for i, n in enumerate(lens):
        qkv[i, :, n:] = 0.0 if pad_value == "zero" else garbage[i, :, n:]
    return qkv, mask, ek, ev


@pytest.mark.parametrize("d,heads,window,t,lens", fma_cases())
def test_fma_attention_against_float64(d, heads, window, t, lens):
    seed = d * 7919 + t * 31 + window
    qkv, mask, ek, ev = fma_inputs(d, heads, window, t, lens, seed, "garbage")
    with _lib.dispatch_log() as log:
        got = run_fma(qkv, mask, heads, window, ek, ev)
    assert log.names == ["attn_fma"]   # <256> for d <= 256, <384> above: the launcher's only rule
    assert not got.isnan().any()
    want = AC.rel_attention(qkv, mask, heads, window, ek, ev)
    f32 = _f32_no_tf32(lambda: AC.rel_attention(qkv, mask, heads, window, ek, ev, dtype=torch.float32))
    # valid query columns, then the padded ones (the uniform rows, which average the +-1e6 of the padded v columns)
    # on their own, so that their scale does not hide the valid columns' error
    assert not AC.attention_failures(got, want, f32, cols=lens)
    for i, n in enumerate(lens):
        if n < t:
            assert not AC.failures(got[i:i + 1, :, n:], want[i:i + 1, :, n:], f32[i:i + 1, :, n:], (1, 2))[0], i
    assert torch.equal(run_fma(qkv, mask, heads, window, ek, ev), got)   # a relaunch is bit-identical
    # contract: valid outputs do not depend on the (finite) padded columns -- bit-identical with zeros there
    zq, _, _, _ = fma_inputs(d, heads, window, t, lens, seed, "zero")
    zero = run_fma(zq, mask, heads, window, ek, ev)
    for i, n in enumerate(lens):
        assert torch.equal(zero[i, :, :n], got[i, :, :n]), i
        if n > 0 and i > 0:   # a ragged row equals its single-row call on its valid columns
            one = run_fma(zq[i:i + 1, :, :n].contiguous(), torch.ones(1, n, device=DEV), heads, window, ek, ev)
            assert torch.equal(one[0], got[i, :, :n]), i


# ------------------------------------------------------------------------------------------------ LayerNorms
LN_C = [1, 7, 8, 9, 192, 384, 385]
LN_T = [1, 31, 32, 33, 300]
# kind 0: (y, mask, eps); kind 1: twice (eps 1e-5, y and mask always)
KIND0 = [(True, True, 1e-5), (False, False, 1e-4), (True, False, 1e-4), (False, True, 1e-5)]


def ln_cases():
    cases = []
    for i, c in enumerate(LN_C):
        for j, t in enumerate(LN_T):
            y, m, eps = KIND0[(i + j) % 4]
            cases.append(pytest.param(0, c, t, y, m, eps, False, id=f"k0_c{c}_t{t}_y{int(y)}_m{int(m)}_eps{eps:g}"))
            twice = bool((i + j) % 2)
            cases.append(pytest.param(1, c, t, True, True, 1e-5, twice, id=f"k1_c{c}_t{t}_twice{int(twice)}"))
    return cases


@pytest.mark.parametrize("kind,c,t,has_y,has_mask,eps,twice", ln_cases())
def test_layernorm_against_float64(kind, c, t, has_y, has_mask, eps, twice):
    g = torch.Generator(device=DEV).manual_seed(c * 131 + t)
    b = 2
    x = torch.randn(b, c, t, generator=g, device=DEV)
    y = torch.randn(b, c, t, generator=g, device=DEV) if has_y else None
    gamma = 1 + 0.5 * torch.randn(c, generator=g, device=DEV)
    beta = 0.1 * torch.randn(c, generator=g, device=DEV)
    if c > 1:   # one column with mean 1e3 and spread 1e-2 (y there stays N(0, 1e-4))
        x[0, :, t // 2] = 1e3 + 1e-2 * torch.randn(c, generator=g, device=DEV)
        if y is not None:
            y[0, :, t // 2] *= 1e-2
    mask = None
    n1 = t // 2
    if has_mask:
        mask = torch.ones(b, t, device=DEV)
        mask[1, n1:] = 0.0
        if kind == 1:   # stale scratch in the masked columns: the select must not let it through
            x[1, :, n1:] = NAN
            y[1, :, n1:] = NAN
    sel = kind == 1
    want = AC.add_layernorm(x, y, gamma, beta, mask, eps=eps, twice=twice, select=sel)
    f32 = AC.add_layernorm(x, y, gamma, beta, mask, eps=eps, twice=twice, select=sel, dtype=torch.float32)
    again = run_ln(kind, x.clone(), y, gamma, beta, mask, eps, twice)
    got = run_ln(kind, x.clone(), y, gamma, beta, mask, eps, twice)
    assert torch.equal(got, again)   # a relaunch is bit-identical
    bad = AC.layernorm_failures(got, want, f32, x, y, gamma, twice)
    assert not bad, bad[:8]
    if has_mask:   # masked columns are exactly 0 (kind 1 over NaN input)
        assert torch.equal(got[1, :, n1:], torch.zeros_like(got[1, :, n1:]))
    # out of place into a NaN-prefilled buffer: every column is written and equals the in-place result
    out = torch.full_like(x, NAN)
    run_ln(kind, x, y, gamma, beta, mask, eps, twice, out=out)
    assert torch.equal(out, got)


# ------------------------------------------------------------------------------------------------ host-side rejections
def _rejected(call):
    n0 = _lib.launch_count()
    rc = call()
    torch.cuda.synchronize()
    assert rc == 1, rc
    assert _lib.launch_count() == n0
    return _lib.lib().b200tts_last_error().decode()


def test_rejections_launch_nothing():
    lib, st = _lib.lib(), _lib.stream_ptr(DEV)
    P = _lib.ptr

    def fma(c, heads, t, window):
        qkv, mask, out = (torch.zeros(1, 3 * c, t, device=DEV), torch.ones(1, t, device=DEV),
                          torch.zeros(1, c, t, device=DEV))
        rel = torch.zeros(max(2 * window + 1, 1), c // max(heads, 1), device=DEV)
        return lambda: lib.b200tts_debug_attention(P(qkv), P(mask), P(rel), P(rel), P(out), 1, c, t, heads, window, st)

    assert "head dim" in _rejected(fma(385, 1, 8, -1))                  # d > 384
    assert "window" in _rejected(fma(96, 1, 8, 16))                     # window > 15
    assert "too long" in _rejected(fma(192, 2, fma_max_t(96, 4) + 1, 4))  # past the shared memory, VITS shape
    assert "too long" in _rejected(fma(384, 1, fma_max_t(384, -1) + 1, -1))
    assert "heads" in _rejected(fma(96, 0, 8, -1))                      # no heads
    qkv, out, lens = torch.zeros(1, 36, 8, device=DEV), torch.zeros(1, 12, 8, device=DEV), torch.full((1,), 8,
                                                                                                   dtype=torch.int32,
                                                                                                   device=DEV)
    assert "d % 8" in _rejected(lambda: lib.b200tts_attention_tc3(P(qkv), P(lens), 1, 12, 1, 8, 8, P(out), st))
    x, y, g, m = (torch.zeros(1, 16, 8, device=DEV), torch.zeros(1, 16, 8, device=DEV), torch.ones(16, device=DEV),
                  torch.ones(1, 8, device=DEV))
    assert "eps" in _rejected(lambda: lib.b200tts_debug_add_layernorm(1, P(x), P(y), 1, P(g), P(g), P(m), P(x), 1, 16, 8,
                                                                      1e-4, st))
    assert "mask" in _rejected(lambda: lib.b200tts_debug_add_layernorm(1, P(x), P(y), 0, P(g), P(g), None, P(x), 1, 16,
                                                                       8, 1e-5, st))
    assert "twice" in _rejected(lambda: lib.b200tts_debug_add_layernorm(0, P(x), P(y), 1, P(g), P(g), None, P(x), 1, 16,
                                                                        8, 1e-5, st))


def test_empty_shapes_launch_nothing():
    lib, st, P = _lib.lib(), _lib.stream_ptr(DEV), _lib.ptr
    t1 = torch.zeros(1, device=DEV)
    n0 = _lib.launch_count()
    for b, t in ((0, 8), (1, 0)):
        assert lib.b200tts_debug_attention(P(t1), P(t1), None, None, P(t1), b, 96, t, 1, -1, st) == 0
        for kind in (0, 1):
            assert lib.b200tts_debug_add_layernorm(kind, P(t1), P(t1), 0, P(t1), P(t1), P(t1), P(t1), b, 16, t, 1e-5,
                                                   st) == 0
    assert lib.b200tts_attention_tc3(P(t1), P(t1), 0, 64, 1, 8, 8, P(t1), st) == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
