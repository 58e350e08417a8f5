"""The attention / LayerNorm checker (attention_check.py) restates the oracle and torch exactly, and rejects the near-miss
mistakes a kernel could make: a relative index off by one, the band's edge dropped, the rel-v terms scaled, padded query
rows zeroed, the unbiased variance, eps outside the root, the `twice` residual dropped, and a mask that multiplies where
it must select.  Each mistake is built from the float64 restatement on CPU tensors at sweep shapes of
test_attention_edges_gpu.py and must break the bound the GPU outputs are held to.
"""
import types

import pytest
import torch
import torch.nn.functional as F

import attention_check as AC
import vits_oracle as O

WINDOW = 4


def _qkv(b, c, t, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(b, 3 * c, t, generator=g), torch.Generator().manual_seed(seed + 1)


def _mask(lens, t):
    return (torch.arange(t)[None, :] < torch.tensor(lens)[:, None]).float()


def _rel(window, d, g):
    return torch.randn(2 * window + 1, d, generator=g), torch.randn(2 * window + 1, d, generator=g)


def _both(fn, *a, **k):
    """(float64, float32) results of one restatement"""
    return fn(*a, **k), fn(*a, **k, dtype=torch.float32)


# T <= window, T = window + 1 and beyond; ragged rows and an all-zero row
REL_CASES = [(2, 3, [3, 0]), (2, 4, [4, 2]), (1, 5, [5, 1]), (2, 9, [9, 6]), (2, 33, [33, 20])]


@pytest.mark.parametrize("heads,t,lens", REL_CASES)
def test_rel_attention_equals_the_oracle(heads, t, lens):
    """identity conv_o; the q / k / v convs of the oracle are applied up front to build the fused q|k|v tensor"""
    c, d = 8 * heads, 8
    g = torch.Generator().manual_seed(t)
    x = torch.randn(len(lens), c, t, generator=g, dtype=torch.float64)
    sd = {f"conv_{s}.weight": torch.randn(c, c, 1, generator=g, dtype=torch.float64) / c ** 0.5 for s in "qkv"}
    sd.update({f"conv_{s}.bias": torch.zeros(c, dtype=torch.float64) for s in "qkvo"})
    sd["conv_o.weight"] = torch.eye(c, dtype=torch.float64)[:, :, None]
    sd["emb_rel_k"] = torch.randn(1, 2 * WINDOW + 1, d, generator=g, dtype=torch.float64)
    sd["emb_rel_v"] = torch.randn(1, 2 * WINDOW + 1, d, generator=g, dtype=torch.float64)
    mask = _mask(lens, t).double()
    attn_mask = mask[:, None, :, None] * mask[:, None, None, :]
    qkv = torch.cat([F.conv1d(x, sd[f"conv_{s}.weight"]) for s in "qkv"], 1)
    for window, ek, ev in ((WINDOW, sd["emb_rel_k"][0], sd["emb_rel_v"][0]), (None, None, None)):
        want = O.rel_attention(sd, x, attn_mask, num_heads=heads, window=window)
        got = AC.rel_attention(qkv, mask, heads, -1 if window is None else window, ek, ev)
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def test_no_window_core_equals_sdpa_on_row_slices():
    b, heads, d, t, lens = 3, 2, 16, 40, [40, 17, 1]
    qkv, _ = _qkv(b, heads * d, t, 3)
    qkv = qkv.double()
    got = AC.rel_attention(qkv, _mask(lens, t), heads)
    got_tc3 = AC.attention_tc3(qkv, lens, heads)
    c = heads * d
    for i, n in enumerate(lens):
        q, k, v = (qkv[i, s * c:(s + 1) * c, :n].reshape(heads, d, n).transpose(1, 2) for s in range(3))
        want = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(c, n)
        torch.testing.assert_close(got[i, :, :n], want, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(got_tc3[i, :, :n], want, rtol=1e-12, atol=1e-12)
        assert float(got_tc3[i, :, n:].abs().sum()) == 0.0


def test_tc3_core_pads_to_the_pitch():
    qkv, _ = _qkv(2, 16, 40, 5)
    out = AC.attention_tc3(qkv, [40, 0], 2)
    assert out.shape == (2, 16, 40) and float(out[1].abs().sum()) == 0.0
    wide = AC.attention_tc3(F.pad(qkv, (0, 60)), [40, 0], 2, pitch=100)
    assert torch.equal(wide[:, :, :40], out) and float(wide[:, :, 40:].abs().sum()) == 0.0


def _shift(e):
    """rel_k / rel_v read one relative index too far: row r holds row r + 1 (zero past the end)"""
    return torch.cat([e[1:], torch.zeros_like(e[:1])])


def _open_band(e):
    """|j - i| < w instead of <= w: the band's two end rows drop out"""
    e = e.clone()
    e[0] = 0
    e[-1] = 0
    return e


# (d, heads, window, t, lens) at shapes of the GPU sweep
REL_MUTANT_SHAPES = [(33, 2, 4, 9, [9, 5]), (96, 2, 4, 65, [65, 40]), (32, 1, 1, 33, [33, 32]), (2, 3, 15, 31, [31, 0])]


@pytest.mark.parametrize("d,heads,window,t,lens", REL_MUTANT_SHAPES)
@pytest.mark.parametrize("mutant", ["index_off_by_one", "band_open", "rel_v_scaled", "padded_rows_zeroed"])
def test_checker_rejects_rel_attention_mutants(d, heads, window, t, lens, mutant):
    qkv, g = _qkv(len(lens), heads * d, t, d + t)
    ek, ev = _rel(window, d, g)
    mask = _mask(lens, t)
    want, f32 = _both(AC.rel_attention, qkv, mask, heads, window, ek, ev)
    assert not AC.attention_failures(f32, want, f32)   # torch's own fp32 passes
    if mutant == "index_off_by_one":
        bad = AC.rel_attention(qkv, mask, heads, window, _shift(ek), _shift(ev))
    elif mutant == "band_open":
        bad = AC.rel_attention(qkv, mask, heads, window, _open_band(ek), _open_band(ev))
    elif mutant == "rel_v_scaled":
        bad = AC.rel_attention(qkv, mask, heads, window, ek, ev / d ** 0.5)
    else:
        bad = want * mask[:, None, :].double()
    assert AC.attention_failures(bad, want, f32), mutant


def test_rel_v_scaling_mutant_is_not_vacuous_at_d_1():
    """d = 1 makes d^-1/2 = 1: the scaled-rel-v mistake is invisible there, so the sweep's d = 1 cases cannot catch it
    and the shapes above must"""
    assert all(s[0] > 1 for s in REL_MUTANT_SHAPES)


def _ln_inputs(b, c, t, seed, offset_col=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, c, t, generator=g) * 0.01
    y = torch.randn(b, c, t, generator=g) * 0.01
    gamma, beta = 1 + 0.5 * torch.randn(c, generator=g), 0.1 * torch.randn(c, generator=g)
    if offset_col and c > 1:   # mean 1e3, spread 1e-2
        x[0, :, t // 2] = 1e3 + 1e-2 * torch.randn(c, generator=g)
    return x, y, gamma, beta


def _duration_predictor_ln():
    """the LayerNorm nested in the oracle's duration_predictor (eps 1e-4), as a function"""
    code = next(k for k in O.duration_predictor.__code__.co_consts if isinstance(k, types.CodeType) and k.co_name == "ln")
    return types.FunctionType(code, vars(O))


def test_layernorm_equals_torch_and_the_oracle():
    x, y, gamma, beta = _ln_inputs(2, 9, 33, 0, offset_col=False)
    x, y = x.double() * 100, y.double() * 100
    mask = _mask([33, 20], 33).double()
    for eps in (1e-4, 1e-5):
        want = F.layer_norm((x + y).transpose(1, 2), (9,), gamma.double(), beta.double(), eps).transpose(1, 2)
        torch.testing.assert_close(AC.add_layernorm(x, y, gamma, beta, eps=eps), want, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(AC.add_layernorm(x, y, gamma, beta, mask, eps=eps), want * mask[:, None],
                                   rtol=1e-12, atol=1e-12)
    ln = _duration_predictor_ln()
    p = {"gamma": gamma.double()[None, :, None], "beta": beta.double()[None, :, None]}
    torch.testing.assert_close(AC.add_layernorm(x, None, gamma, beta, eps=1e-4), ln(p, x), rtol=1e-12, atol=1e-12)
    # kind 1: (x + y) + y, then a select that is exact 0 even over NaN
    xn = x.clone()
    xn[1, :, 20:] = float("nan")
    got = AC.add_layernorm(xn, y, gamma, beta, mask, eps=1e-5, twice=True, select=True)
    want = F.layer_norm((x + 2 * y).transpose(1, 2), (9,), gamma.double(), beta.double(), 1e-5).transpose(1, 2)
    torch.testing.assert_close(got[0], want[0], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(got[1, :, :20], want[1, :, :20], rtol=1e-12, atol=1e-12)
    assert torch.equal(got[1, :, 20:], torch.zeros_like(got[1, :, 20:]))


def _ln_mutant(x, y, gamma, beta, mask, eps, mutant):
    v = x.double() + y.double()
    if mutant != "twice_dropped":
        v = v + y.double()          # the checked kernel is kind 1 with twice
    mean = v.mean(1, keepdim=True)
    var = (v - mean).pow(2).mean(1, keepdim=True)
    if mutant == "unbiased_variance":
        var = var * v.shape[1] / (v.shape[1] - 1)
    denom = torch.sqrt(var) + eps if mutant == "eps_outside_root" else torch.sqrt(var + eps)
    out = (v - mean) / denom * gamma.double()[None, :, None] + beta.double()[None, :, None]
    m = mask.double()[:, None, :]
    if mutant == "mask_multiplies":
        return out * m
    return torch.where(m != 0, out, torch.zeros_like(out))


@pytest.mark.parametrize("c,t", [(7, 31), (9, 33), (192, 32), (384, 300), (385, 33)])
@pytest.mark.parametrize("mutant", ["unbiased_variance", "eps_outside_root", "twice_dropped", "mask_multiplies"])
def test_checker_rejects_layernorm_mutants(c, t, mutant):
    x, y, gamma, beta = _ln_inputs(2, c, t, c + t)
    mask = _mask([t, t // 2], t)
    x[1, :, t // 2:] = float("nan")    # stale scratch in the masked columns of kind 1
    kw = dict(eps=1e-5, twice=True, select=True)
    want, f32 = _both(AC.add_layernorm, x, y, gamma, beta, mask, **kw)
    assert not AC.layernorm_failures(f32, want, f32, x, y, gamma, twice=True)
    bad = _ln_mutant(x, y, gamma, beta, mask, 1e-5, mutant)
    assert AC.layernorm_failures(bad, want, f32, x, y, gamma, twice=True), mutant


def test_one_pass_variance_fails_the_offset_column():
    """the offset column's own allowance is loose (its fp32 mean is only good to ~1e-5 of 1e3), but not so loose that a
    one-pass variance passes"""
    c, t = 384, 33
    x, y, gamma, beta = _ln_inputs(1, c, t, 7)
    want, f32 = _both(AC.add_layernorm, x, None, gamma, beta, eps=1e-5)
    v = x.float()
    mean = v.mean(1, keepdim=True)
    var = (v * v).mean(1, keepdim=True) - mean * mean          # E[v^2] - mean^2 in fp32
    bad = (v - mean) * torch.rsqrt(var + 1e-5) * gamma[None, :, None] + beta[None, :, None]
    assert (0, t // 2) in AC.layernorm_failures(bad, want, f32, x, None, gamma)
    assert not AC.layernorm_failures(f32, want, f32, x, None, gamma)
