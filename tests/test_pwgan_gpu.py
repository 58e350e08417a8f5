"""Parallel WaveGAN on the GPU: the upsampler tables against the float64 stage chain (every edge sample), each fused
residual layer alone against float64 (every dilation, NaN around and past every tensor, no store outside the output
rows), the whole generator against the oracle (tests/pwgan_oracle.py, itself pinned to the reference) on supplied and on
seeded noise, determinism with a NaN-poisoned workspace, the pinned dispatch, the split-fp16 range flag and the
Glow-TTS -> GAN chain."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import conv_check
import glow_oracle as GO
import pwgan_oracle as PO
from ref_golden import layout, seeded_state_dict
from test_glow_oracle_cpu import run_case
from tts_b200 import _lib
from tts_b200.pwgan import ParallelWaveganGenerator

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WAVE_REL_TOL = 1e-4


def rel_rms(got, want):
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def gpu_model(seed=5, **over):
    m = ParallelWaveganGenerator(**over).eval()
    sd = seeded_state_dict(layout(m.state_dict()), seed)
    m.load_state_dict(sd)
    return m.to(DEV), sd


def kw(m):
    return dict(upsample_factors=tuple(m.upsample_factors), num_res_blocks=m.num_res_blocks, stacks=m.stacks)


def want_inference(m, sd, c, noise):
    """The oracle in float64 on the GPU (the reference's sum order, no tensor-core rounding)."""
    sd64 = {k: v.to(DEV).double() for k, v in sd.items()}
    return PO.inference(sd64, c.to(DEV).double(), noise.to(DEV).double(), **kw(m)).float()


@pytest.mark.parametrize("factors", [(4, 4, 4, 4), (3, 5, 4)])
@pytest.mark.parametrize("frames", [5, 6, 7, 64])
def test_upsampler_tables_against_float64_chain(factors, frames):
    m, sd = gpu_model(upsample_factors=list(factors))
    assert m.min_frames(DEV) <= 5
    a = torch.randn(16, frames, generator=torch.Generator().manual_seed(frames)).to(DEV)
    got = m.upsample(a).double()
    want = PO.stages({k: v.to(DEV).double() for k, v in sd.items()}, a.double().unsqueeze(0), factors)[0]
    assert got.shape == want.shape
    err = (got - want).abs().max() / want.abs().max()
    assert err <= 1e-6, float(err)
    # every edge sample (two frames' worth at each end) on its own
    hop = m.upsample_scale
    for sl in (slice(0, 2 * hop), slice(-2 * hop, None)):
        e = (got[:, sl] - want[:, sl]).abs().max() / want[:, sl].abs().max()
        assert e <= 1e-6, (sl, float(e))


CASES = {
    "default_T1": (dict(), 1),
    "default_T3": (dict(), 3),
    "default_T40": (dict(), 40),
    "factors_3_5_4": (dict(upsample_factors=[3, 5, 4]), 7),
    "stacks_2_blocks_20": (dict(stacks=2, num_res_blocks=20), 9),
}


@pytest.mark.parametrize("case", list(CASES))
def test_generator_against_oracle(case):
    over, t = CASES[case]
    m, sd = gpu_model(**over)
    g = torch.Generator().manual_seed(3)
    c = torch.randn(2, 80, t, generator=g)
    noise = torch.randn(2, 1, (t + 4) * m.upsample_scale, generator=g)
    got = m.inference(c.to(DEV), noise=noise)
    want = want_inference(m, sd, c, noise)
    assert got.shape == want.shape == (2, 1, (t + 4) * m.upsample_scale)
    assert rel_rms(got, want) <= WAVE_REL_TOL, rel_rms(got, want)
    # forward (no pad) on a long enough input
    c2 = torch.randn(1, 80, 6, generator=g)
    n2 = torch.randn(1, 1, 6 * m.upsample_scale, generator=g)
    want2 = PO.generator({k: v.to(DEV).double() for k, v in sd.items()}, c2.to(DEV).double(), n2.to(DEV).double(),
                         **kw(m)).float()
    assert rel_rms(m(c2.to(DEV), noise=n2), want2) <= WAVE_REL_TOL


def test_forward_shorter_than_min_frames_raises():
    """forward(c) without the pad takes T >= min_frames (the upsampler tables' shortest exact length); inference pads
    first, so T = 1 runs there (test_generator_against_oracle)."""
    m, _ = gpu_model()
    t_min = m.min_frames(DEV)
    assert 1 <= t_min <= 5
    if t_min > 1:
        with pytest.raises(RuntimeError, match="need at least"):
            m(torch.randn(1, 80, t_min - 1, device=DEV), noise=torch.randn(1, 1, (t_min - 1) * 256))
    assert m(torch.randn(1, 80, t_min, device=DEV), noise=torch.randn(1, 1, t_min * 256)).shape == (1, 1, t_min * 256)


def test_bench_shape_against_oracle():
    """The MelGAN bench batch: 32 utterances of 384 frames, inference (388 frames after the pad)."""
    m, sd = gpu_model(seed=11)
    g = torch.Generator().manual_seed(4)
    c = torch.randn(32, 80, 384, generator=g)
    noise = torch.randn(32, 1, 388 * 256, generator=g)
    got = m.inference(c.to(DEV), noise=noise)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd32 = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        want = PO.inference(sd32, c.to(DEV), noise.to(DEV), **kw(m))
    assert rel_rms(got, want) <= WAVE_REL_TOL, rel_rms(got, want)


def test_seeded_draw_matches_oracle():
    m, sd = gpu_model(seed=6)
    c = torch.randn(2, 80, 5, generator=torch.Generator().manual_seed(8))
    torch.manual_seed(1234)
    got = m.inference(c.to(DEV))
    torch.manual_seed(1234)
    noise = torch.randn([2, 1, 9 * 256])
    assert rel_rms(got, want_inference(m, sd, c, noise)) <= WAVE_REL_TOL


def test_determinism_poisoned_workspace_and_dispatch():
    m, _ = gpu_model(seed=7)
    c = torch.randn(3, 80, 20, generator=torch.Generator().manual_seed(9)).to(DEV)
    noise = torch.randn(3, 1, 24 * 256, generator=torch.Generator().manual_seed(10))
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with _lib.dispatch_log() as log:
        a = m.inference(c, noise=noise)
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    b = m.inference(c, noise=noise)
    for buf in _lib._workspaces.values():
        buf.view(torch.float32)[: buf.numel() // 4].fill_(float("nan"))
    cc = m.inference(c, noise=noise)
    assert torch.equal(a, b) and torch.equal(a, cc) and torch.isfinite(a).all()
    # the folded conditioning conv, one fused launch per residual layer (dilations 1 .. 512), the 64 -> 64 tail conv on
    # the tensor cores and the 64 -> 1 conv on the FMA kernel; plus first_conv, which the dispatch log does not list
    assert log.names[:31] == ["pwgan_aux"] + ["pwgan_tc"] * 30, log.names
    assert log.names[31] in ("tc3", "tc3_grouped") and log.names[32:] == ["fma"], log.names
    assert launches == 34, launches


def test_range_flag_fails_loudly_once():
    """A first_conv scaled far beyond fp16's range: the first residual layer reads |x| > 65504 and the error surfaces
    once, through the conv engine's range flag; later calls run normally."""
    m, sd = gpu_model(seed=8, num_res_blocks=3, stacks=1)
    good = ParallelWaveganGenerator(num_res_blocks=3, stacks=1).eval()
    good.load_state_dict(sd)
    good.to(DEV)
    with torch.no_grad():
        m.first_conv.parametrizations.weight.original0.mul_(1e7)
    m.repack()
    c = torch.randn(1, 80, 6, device=DEV)
    noise = torch.randn(1, 1, 10 * 256)
    errors = 0
    for net in (m, good, good):
        try:
            net.inference(c, noise=noise)
            torch.cuda.synchronize()
        except RuntimeError as e:
            assert "65504" in str(e), str(e)
            errors += 1
    assert errors == 1


def test_glow_tts_to_parallel_wavegan_chain():
    """GlowTTS -> vocoder_input(padding=2) -> GAN(ParallelWaveganConfig()).model_g.forward, against the oracle chain."""
    from tts_b200.glow_tts import GlowTTS
    from tts_b200.vocoder import GAN, AudioNorm, ParallelWaveganConfig, vocoder_input
    cfg, sd, x, lens, extra, noise = run_case("default")
    want_mel = GO.inference(sd, x, lens, cfg)["model_outputs"]
    gan = GAN(ParallelWaveganConfig()).eval()
    gsd = seeded_state_dict(layout(gan.model_g.state_dict()), 13)
    gan.model_g.load_state_dict(gsd)
    gan.to(DEV)
    glow = GlowTTS(cfg).eval()
    glow.load_state_dict(sd)
    mel = glow.to(DEV).inference(x.to(DEV), {"x_lengths": lens.to(DEV)})["model_outputs"]
    t = mel.shape[1]
    wn = torch.randn(mel.shape[0], 1, (t + 4) * 256, generator=torch.Generator().manual_seed(2))
    want = want_inference(gan.model_g, gsd, want_mel.transpose(1, 2), wn)
    voc_in = vocoder_input(mel, AudioNorm.identity(), AudioNorm.identity(), padding=2, time_last=False)
    assert rel_rms(gan.model_g.forward(voc_in, noise=wn), want) <= WAVE_REL_TOL
    assert rel_rms(gan.model_g.inference(mel.transpose(1, 2), noise=wn), want) <= WAVE_REL_TOL


# ---------------------------------------------------------------------------------------------- one fused layer alone
LAYER_REL_TOL = 5e-5
_MODELS = {}


def layer_model(factors):
    if factors not in _MODELS:
        _MODELS[factors] = gpu_model(seed=21, upsample_factors=list(factors))
    return _MODELS[factors]


def want_layer(sd64, layer, mel, x, skip, factors, num_res_blocks=30, per_stack=10):
    """ResidualBlock.forward and the generator's skip sum for one layer, in float64."""
    p = f"conv_layers.{layer}."
    d = 2 ** (layer % per_stack)
    h = F.conv1d(x, PO.conv_weight(sd64, p + "conv"), sd64[p + "conv.bias"], padding=d, dilation=d)
    xa, xb = h.split(64, dim=1)
    a = F.conv1d(PO.upsample(sd64, mel, factors), PO.conv_weight(sd64, p + "conv1x1_aux"))
    ca, cb = a.split(64, dim=1)
    z = torch.tanh(xa + ca) * torch.sigmoid(xb + cb)
    s = F.conv1d(z, PO.conv_weight(sd64, p + "conv1x1_skip"), sd64[p + "conv1x1_skip.bias"])
    x_new = (F.conv1d(z, PO.conv_weight(sd64, p + "conv1x1_out"), sd64[p + "conv1x1_out.bias"]) + x) * 0.25
    skip_new = s if layer == 0 else skip + s
    if layer == num_res_blocks - 1:
        skip_new = skip_new * math.sqrt(1.0 / num_res_blocks)
    return x_new, skip_new


def guarded(b, pitch, guard):
    """A [b, 64, pitch] view in the middle of a NaN-filled store with `guard` floats before and after it."""
    store = torch.full((2 * guard + b * 64 * pitch,), float("nan"), device=DEV)
    return store, store[guard: guard + b * 64 * pitch].view(b, 64, pitch)


def bits(t):
    return t.contiguous().view(torch.int32).clone()


@pytest.mark.parametrize("factors,frames", [((4, 4, 4, 4), 5), ((4, 4, 4, 4), 64), ((3, 5, 4), 5), ((3, 5, 4), 7)])
@pytest.mark.parametrize("layer", list(range(10)) + [29])
def test_fused_layer_against_float64(factors, frames, layer):
    """One residual layer (dilations 1 .. 512 of the first stack; layer 0 stores the skip sum, layer 29 -- dilation 512 --
    also scales it) against float64, with NaN past every row, in the whole output buffer and around every tensor: the
    layer reads none of it and writes nothing outside its output rows.  (3, 5, 4) gives rows of 300 and 420 samples,
    not a multiple of the 128-column tile."""
    m, sd = layer_model(factors)
    hop = m.upsample_scale
    ts = frames * hop
    pitch = (ts + 3) // 4 * 4 + 4
    guard, b = 1024, 2
    g = torch.Generator().manual_seed(100 * layer + frames)
    mel = torch.randn(b, 80, frames, generator=g)
    x_val = torch.randn(b, 64, ts, generator=g)
    skip_val = torch.randn(b, 64, ts, generator=g)
    xs, x = guarded(b, pitch, guard)
    ss, skip = guarded(b, pitch, guard)
    ns, x_new = guarded(b, pitch, guard)            # the ping-pong buffer: NaN everywhere
    x[:, :, :ts] = x_val.to(DEV)
    if layer > 0:                                   # layer 0 stores the skip sum: its old content must not be read
        skip[:, :, :ts] = skip_val.to(DEV)
    x_bits, skip_tail, new_tail = bits(xs), bits(skip[:, :, ts:]), bits(x_new[:, :, ts:])
    ss_head, ss_tail = bits(ss[:guard]), bits(ss[-guard:])
    ns_head, ns_tail = bits(ns[:guard]), bits(ns[-guard:])
    L = _lib.lib()
    h = m._ensure_handle(DEV)
    ws = torch.full((L.b200tts_pwgan_workspace_bytes(h, b, frames) // 4,), float("nan"), device=DEV)
    mel_d = mel.to(DEV).contiguous()
    with _lib.dispatch_log() as log:
        rc = L.b200tts_pwgan_layer(h, layer, _lib.ptr(mel_d), b, frames, 0, _lib.ptr(x), _lib.ptr(skip), _lib.ptr(x_new),
                                   pitch, _lib.ptr(ws), ctypes.c_size_t(ws.numel() * 4), _lib.stream_ptr(DEV))
    torch.cuda.synchronize()
    _lib.check(rc, "pwgan_layer")
    assert log.names == ["pwgan_aux", "pwgan_tc"], log.names
    sd64 = {k: v.to(DEV).double() for k, v in sd.items()}
    want_x, want_s = want_layer(sd64, layer, mel_d.double(), x_val.to(DEV).double(),
                                skip_val.to(DEV).double() if layer > 0 else None, factors)
    for name, got, want in (("x_new", x_new[:, :, :ts], want_x), ("skip", skip[:, :, :ts], want_s)):
        bad, meas = conv_check.failures(got, want, LAYER_REL_TOL)
        assert not bad, (name, bad, meas)
    # nothing outside the output rows was written; x was not written at all
    assert torch.equal(bits(xs), x_bits)
    assert torch.equal(bits(skip[:, :, ts:]), skip_tail) and torch.equal(bits(x_new[:, :, ts:]), new_tail)
    assert torch.equal(bits(ss[:guard]), ss_head) and torch.equal(bits(ss[-guard:]), ss_tail)
    assert torch.equal(bits(ns[:guard]), ns_head) and torch.equal(bits(ns[-guard:]), ns_tail)
