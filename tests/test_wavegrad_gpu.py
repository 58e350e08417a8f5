"""WaveGrad on the GPU (``-m gpu``): each new conv variant on its own against float64 at the default config's layer
shapes (NaN past every row), ``Wavegrad.forward`` against float64, ``inference`` against the fp32 oracle with supplied
noise and with the reference's own draws, positional-encoding tables reused across lengths, determinism over a
NaN-filled workspace, the dispatch of every layer and the launches per refinement step."""
import numpy as np
import torch.nn.functional as F
import pytest
import torch

import wavegrad_oracle as WO
from ref_golden import layout, seeded_state_dict
from tts_b200 import _lib
from tts_b200 import wavegrad as W
from tts_b200.conv import FusedConv1d

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
SMALL = dict(in_channels=16, y_conv_channels=8, x_conv_channels=32, dblock_out_channels=[16, 16],
             ublock_out_channels=[32, 16, 16], upsample_factors=[3, 2, 2], upsample_dilations=[[1, 2, 1, 2]] * 3)


def model(over=None, steps=50, seed=5):
    cfg = W.WavegradConfig(model_params=W.WavegradArgs(**(over or {})))
    cfg.test_noise_schedule = {"min_val": 1e-6, "max_val": 1e-2, "num_steps": steps}
    m = W.Wavegrad(cfg).eval()
    sd = seeded_state_dict(layout(m.state_dict()), seed)
    m.load_state_dict(sd)
    s = cfg.test_noise_schedule
    m.compute_noise_level(np.linspace(s["min_val"], s["max_val"], s["num_steps"]))
    return m.to(DEV), sd, cfg


def rel_rms(got, want):
    got, want = got.double().cpu(), want.double().cpu()
    return ((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt()).item()


def sd64(sd):
    return {k: v.double().to(DEV) for k, v in sd.items()}


@pytest.fixture(autouse=True)
def _fp32_eager():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("over,T", [(None, 1), (None, 7), (None, 40), (SMALL, 5), (SMALL, 70)])
def test_forward_matches_float64(over, T):
    """Every conv mode at the default shapes: T = 1 and 7 run the short stages on the FMA tile kernel, T = 40 puts every
    stage but x_conv on the tensor cores (resampled inputs, FiLM epilogues); T = 7 is not a multiple of 4."""
    m, sd, cfg = model(over)
    g = torch.Generator().manual_seed(T)
    spec = torch.randn(2, cfg.model_params.in_channels, T, generator=g)
    y = torch.randn(2, 1, m.hop_len * T, generator=g)
    ns = torch.rand(2, generator=g)
    got = m(y.to(DEV), spec.to(DEV), ns.to(DEV))
    want = WO.forward(sd64(sd), y.double().to(DEV), spec.double().to(DEV), ns.double().to(DEV), cfg.model_params)
    assert got.shape == y.shape
    assert rel_rms(got, want) <= 1e-5


def test_inference_supplied_noise_matches_oracle():
    m, sd, cfg = model()
    n_steps = len(m.alpha)
    g = torch.Generator().manual_seed(2)
    spec = torch.randn(2, 80, 8, generator=g)
    y0 = torch.randn(2, 1, 8 * m.hop_len, generator=g)
    zs = torch.randn(n_steps - 1, 2, 1, 8 * m.hop_len, generator=g)
    got = m.inference(spec.to(DEV), init_noise=y0.to(DEV), step_noise=zs.to(DEV))
    sched = WO.schedule(np.linspace(1e-6, 1e-2, n_steps))
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    want = WO.inference(sdd, spec.to(DEV), sched, cfg.model_params, init_noise=y0.to(DEV), step_noise=zs.to(DEV))
    assert rel_rms(got, want) <= 1e-5
    inside = (got.abs() < 1).float().mean().item()
    assert inside > 0.9, inside          # a clamped sample hides no error: most must be strictly inside (-1, 1)


def test_inference_draws_match_reference_order():
    """No noise supplied: the initial signal on the CPU generator, one randn_like per step on the device generator --
    the oracle run eagerly on the same GPU with the reference's draw order gives the same waveform."""
    m, sd, cfg = model(steps=6)
    spec = torch.randn(1, 80, 6, generator=torch.Generator().manual_seed(4)).to(DEV)
    torch.manual_seed(123)
    got = m.inference(spec)
    torch.manual_seed(123)
    want = WO.inference({k: v.to(DEV) for k, v in sd.items()}, spec, WO.schedule(np.linspace(1e-6, 1e-2, 6)),
                        cfg.model_params)
    assert rel_rms(got, want) <= 1e-5


def test_repeat_and_nan_workspace_are_bit_identical():
    m, _, _ = model(steps=4)
    spec = torch.randn(2, 80, 37, generator=torch.Generator().manual_seed(6)).to(DEV)
    y0 = torch.randn(2, 1, 37 * m.hop_len, generator=torch.Generator().manual_seed(7)).to(DEV)
    zs = torch.randn(3, 2, 1, 37 * m.hop_len, generator=torch.Generator().manual_seed(8)).to(DEV)
    a = m.inference(spec, init_noise=y0, step_noise=zs)
    b = m.inference(spec, init_noise=y0, step_noise=zs)
    for buf in _lib._workspaces.values():
        buf.view(torch.float32).fill_(float("nan"))
    c = m.inference(spec, init_noise=y0, step_noise=zs)
    assert torch.equal(a, b) and torch.equal(a, c) and not torch.isnan(a).any()


MIXED = dict(in_channels=80, y_conv_channels=40, x_conv_channels=96, dblock_out_channels=[64, 64],
             ublock_out_channels=[48, 64, 64], upsample_factors=[4, 2, 2], upsample_dilations=[[1, 2, 1, 2]] * 3)


def expected_dispatch(p, T):
    """The kernel every conv of one inference should take: x_conv, then per step y_conv, FiLMs, DBlocks, UBlocks."""
    def kind(rows, cin, L, wg=False, near=False, dil=1):
        if L < 128 or rows < 32 or cin < 8:                      # short stages / narrow layers: the FMA tile kernel
            return ("fma_wg" + ("_near" if near else "")) if wg else "fma"
        prec = "f16x3" if cin % 16 == 0 else "tf32"             # split-fp16 where Cin % 16 == 0, else 3xTF32
        if wg:
            return f"tc3w_{prec}" + ("_near" if near else "")
        if rows in (32, 64) and L >= 256 and (128 // rows - 1) * dil <= 15:
            return "tc3_grouped"
        return "tc3"

    f, n = p.upsample_factors, len(p.upsample_factors)
    L = [int(np.prod(f)) * T]
    for df in reversed(f[1:]):
        L.append(L[-1] // df)
    step = ["fma"]                                               # y_conv: one input channel
    ic = p.y_conv_channels
    for i in range(n):
        oc = p.ublock_out_channels[n - 1 - i]
        step += [kind(ic, ic, L[i], wg=True), kind(2 * oc, ic, L[i])]
        if i + 1 < n:
            d, Ld = p.dblock_out_channels[i], L[i + 1]
            step += [kind(d, ic, Ld, True, True), kind(d, ic, Ld, True, True), kind(d, d, Ld, dil=2), kind(d, d, Ld, dil=4)]
            ic = d
    xc = p.x_conv_channels
    for u in range(n):
        h, Lu, dl = p.ublock_out_channels[u], L[n - 1 - u], p.upsample_dilations[u]
        step += [kind(h, xc, Lu, True, True), kind(h, xc, Lu, True, True), kind(h, h, Lu, True), kind(h, h, Lu, True),
                 kind(h, h, Lu, dil=dl[3])]
        xc = h
    return [kind(p.x_conv_channels, p.in_channels, T)], step


@pytest.mark.parametrize("over,T", [(None, 128), (None, 1), (MIXED, 32)])
def test_dispatch_and_launches_per_step(over, T):
    """Every layer's kernel: the WaveGrad tensor-core variant by operand type (split-fp16 for Cin % 16 == 0, else
    3xTF32) and input mode (nearest-resampled or not), the plain / grouped kernels for the other layers, and the FMA
    variants for the stages shorter than a tensor-core tile (T = 1)."""
    m, _, cfg = model(over, steps=3)
    spec = torch.randn(1, cfg.model_params.in_channels, T, generator=torch.Generator().manual_seed(9)).to(DEV)
    m.inference(spec)                      # handle, tables and workspace in place
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with _lib.dispatch_log() as log:
        m.inference(spec)
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    first, step = expected_dispatch(cfg.model_params, T)
    got = log.names
    assert got[:1] == first and len(got) == 1 + 3 * len(step), got[:1]
    for i, (g_, w_) in enumerate(zip(got[1:1 + len(step)], step)):
        assert g_ == w_, (i, g_, w_)
    assert got == first + 3 * step
    assert launches == 1 + 3 * (len(step) + 1)             # x_conv once per inference; out_conv is the engine's own
    if over is None:
        assert len(step) + 1 == 53
    if over is None and T == 128:
        assert set(step[1:]) == {"tc3", "tc3w_f16x3", "tc3w_f16x3_near"}
    if over is MIXED:
        assert "tc3w_tf32" in step and "tc3w_tf32_near" in step and "tc3_grouped" in step


# ---- each WaveGrad conv variant on its own, against float64, with NaN past every row it must not read or write
def _nan_rows(t, length, pitch):
    out = torch.full(t.shape[:-1] + (pitch,), float("nan"), dtype=torch.float32, device=DEV)
    out[..., :length] = t[..., :length]
    return out


# name -> (Cout, Cin, K, dilation, source columns, conv columns (resampled when they differ), input slope, options)
LAYERS = {
    "ublock0_main0_up4": (512, 768, 3, 1, 37, 148, 0.2, dict(film=True, y2=True)),
    "ublock_main1_res2": (128, 128, 3, 2, 131, 131, 0.2, dict(film=True, res="inplace")),
    "ublock_main0_up3": (256, 512, 3, 1, 43, 129, 0.2, dict(film=True)),
    "dblock_main0_down4": (256, 128, 3, 1, 1028, 257, 0.2, dict()),
    "dblock_res_down4": (256, 128, 1, 1, 1028, 257, 1.0, dict()),
    "film_input": (128, 128, 3, 1, 257, 257, 1.0, dict(lrelu=True, add=True, res="pe")),
}


@pytest.mark.parametrize("kernel", ["f16x3", "tf32x3", "fma"])
@pytest.mark.parametrize("name", list(LAYERS))
def test_wavegrad_conv_variant_matches_float64(name, kernel):
    cout, cin, k, dil, src, tin, slope, o = LAYERS[name]
    B = 2
    g = torch.Generator().manual_seed(len(name))
    w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    conv = FusedConv1d(w, b, dilation=dil, padding=dil * (k - 1) // 2, tensor_cores=kernel != "fma",
                       precision="fp32" if kernel == "fma" else kernel)
    near = tin != src
    xs = torch.randn(B, cin, src, generator=g)
    X = _nan_rows(xs.to(DEV), src, (src + 3) // 4 * 4 + 4)
    tout, pitch = tin, (tin + 3) // 4 * 4 + 4
    Y = torch.full((B, cout, pitch), float("nan"), device=DEV)
    add = (torch.randn(B, generator=g) * 0.5).to(DEV) if o.get("add") else None
    res = res_bs = res_cs = None
    if o.get("res") == "pe":                                   # batch stride 0, a pitch longer than the row
        lp = tout + 37
        res, res_bs, res_cs = (torch.randn(cout, lp, generator=g) * 2e-4).to(DEV), 0, lp
    elif o.get("res") == "inplace":                            # res2 = R + conv, written back into R (y2 aliases R)
        res = _nan_rows(torch.randn(B, cout, tout, generator=g).to(DEV), tout, pitch)
        res_bs, res_cs = cout * pitch, pitch
    res_in = None if res is None else res.clone()
    Y2 = res if o.get("res") == "inplace" else (torch.full_like(Y, float("nan")) if o.get("y2") else None)
    film = _nan_rows(torch.randn(B, 2 * cout, tout, generator=g).to(DEV), tout, pitch) if o.get("film") else None
    h = conv._handle(DEV)
    with _lib.dispatch_log() as log:
        rc = _lib.lib().b200tts_conv1d_forward_wavegrad(
            h, _lib.ptr(X), cin * X.shape[-1], X.shape[-1], B, tin, src if near else 0, slope, int(bool(o.get("lrelu"))),
            _lib.ptr(add), _lib.ptr(res), res_bs or 0, res_cs or 0, _lib.ptr(film), 2 * cout * pitch, pitch, cout,
            _lib.ptr(Y), cout * pitch, pitch, _lib.ptr(Y2), _lib.stream_ptr(DEV))
        torch.cuda.synchronize()
    _lib.check(rc, "conv1d_forward_wavegrad")
    want_kind = {"f16x3": "tc3w_f16x3", "tf32x3": "tc3w_tf32", "fma": "fma_wg"}[kernel] + ("_near" if near else "")
    assert log.names == [want_kind]
    # float64
    x64 = xs.double().to(DEV)
    if near:
        x64 = F.interpolate(x64, size=tin)
    u = F.conv1d(F.leaky_relu(x64, slope), w.double().to(DEV), b.double().to(DEV), padding=dil * (k - 1) // 2,
                 dilation=dil)
    if o.get("lrelu"):
        u = F.leaky_relu(u, 0.2)
    if add is not None:
        u = u + add.double()[:, None, None]
    if o.get("res") == "pe":
        u = u + res.double()[None, :, :tout]
    elif res_in is not None:
        u = u + res_in.double()[..., :tout]
    pre = u
    if film is not None:
        fd = film.double()
        u = fd[:, :cout, :tout] + fd[:, cout:, :tout] * u
    # one layer with up to 2 304 products per output: the per-layer bound of the MelGAN / HiFiGAN layer tests
    assert rel_rms(Y[..., :tout], u) <= 5e-5
    assert torch.isnan(Y[..., tout:]).all() and not torch.isnan(Y[..., :tout]).any()   # nothing stored past the row
    if Y2 is not None:
        assert rel_rms(Y2[..., :tout], pre) <= 5e-5
        assert torch.isnan(Y2[..., tout:]).all()


def test_pe_tables_reused_for_shorter_inputs():
    """The tables grow to the longest input and serve shorter ones through their pitch: results stay right, and a
    sequence of lengths allocates no new tables past the longest."""
    m, sd, cfg = model()
    g = torch.Generator().manual_seed(12)
    ptr = None
    for T in (12, 5, 9, 12, 3):
        spec = torch.randn(1, 80, T, generator=g)
        y = torch.randn(1, 1, m.hop_len * T, generator=g)
        ns = torch.rand(1, generator=g)
        got = m(y.to(DEV), spec.to(DEV), ns.to(DEV))
        want = WO.forward(sd64(sd), y.double().to(DEV), spec.double().to(DEV), ns.double().to(DEV), cfg.model_params)
        assert rel_rms(got, want) <= 1e-5, T
        assert m._pe[1] == 12
        ptr = ptr or [t.data_ptr() for t in m._pe[2]]
        assert [t.data_ptr() for t in m._pe[2]] == ptr          # built once, at the first (longest) length


def test_mel_from_text_to_wavegrad():
    """A vocoder_input hand-off into WaveGrad, as Synthesizer calls it ([1, C, T])."""
    from tts_b200.vocoder import AudioNorm, vocoder_input
    m, sd, cfg = model(steps=3)
    mel = (torch.rand(1, 21, 80, generator=torch.Generator().manual_seed(3)) * 8 - 4).to(DEV)   # [B, T, C] model output
    x = vocoder_input(mel, AudioNorm(), AudioNorm(), time_last=False)
    torch.manual_seed(5)
    got = m.inference(x)
    torch.manual_seed(5)
    want = WO.inference({k: v.to(DEV) for k, v in sd.items()}, x.contiguous(), WO.schedule(np.linspace(1e-6, 1e-2, 3)),
                        cfg.model_params)
    assert got.shape == (1, 1, 21 * 256) and rel_rms(got, want) <= 1e-5
