"""MelGAN generators on the GPU: every reflect-padded layer shape of the three default generators against a float64
``nn.Conv1d(padding_mode="reflect")`` (all four row-length residues, the shortest legal row, a many-tile launch, an
all-edge-tile launch, a NaN tail past the row that must never be read), the pinned dispatch, PQMF synthesis, the
generators against the CPU oracle (tests/melgan_oracle.py, itself pinned to the reference), bit-identical repeat runs
and the Glow-TTS -> multi-band MelGAN chain."""
import pytest
import torch
import torch.nn.functional as F

import glow_oracle as GO
import melgan_oracle as MO
from lowp_reference import lowp_conv1d
from test_glow_oracle_cpu import run_case
from test_melgan_oracle_cpu import CASES, build_case, oracle_kwargs
from tts_b200 import _lib
from tts_b200.conv import FusedConv1d
from tts_b200.melgan import PQMF, MultibandMelganGenerator

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def rel_rms(got, want):
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def rms(got, want):
    return float((got - want).pow(2).mean().sqrt())


# every reflect-padded layer shape of the default generators (plain / full-band: base 512, multi-band: base 384):
# name -> (Cin, Cout, K, dilation, input slope, tanh epilogue, dispatch of an aligned long row)
LAYERS = {
    "pre512_k7": (80, 512, 7, 1, 1.0, False, "tc3"),
    "pre384_k7": (80, 384, 7, 1, 1.0, False, "tc3"),
    "res256_d1": (256, 256, 3, 1, 0.2, False, "tc3"),
    "res192_d3": (192, 192, 3, 3, 0.2, False, "tc3"),
    "res128_d9": (128, 128, 3, 9, 0.2, False, "tc3"),
    "res96_d27": (96, 96, 3, 27, 0.2, False, "tc3"),
    "res64_d3": (64, 64, 3, 3, 0.2, False, "tc3_grouped"),
    "res64_d9": (64, 64, 3, 9, 0.2, False, "tc3_grouped"),
    "res64_d27": (64, 64, 3, 27, 0.2, False, "tc3"),
    "res48_d1": (48, 48, 3, 1, 0.2, False, "tc3"),
    "res32_d1": (32, 32, 3, 1, 0.2, False, "tc3_grouped"),
    "res32_d27": (32, 32, 3, 27, 0.2, False, "tc3"),
    "post1_k7": (32, 1, 7, 1, 0.2, True, "row1"),
    "post4_k7": (48, 4, 7, 1, 0.2, True, "fma"),
}


def layer(name, precision="fp32"):
    cin, cout, k, d, slope, tanh, _ = LAYERS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    w = (torch.rand(cout, cin, k, generator=g) * 2 - 1) / (cin * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.05
    conv = FusedConv1d(w, b, dilation=d, padding=(k - 1) // 2 * d, padding_mode="reflect", precision=precision)
    return conv, w, b, slope, tanh


def padded_view(x, tail):
    """x [B, C, T] as a view whose row pitch is T rounded up to 4 plus 4, the columns past T filled with `tail`."""
    b, c, t = x.shape
    store = torch.full((b, c, (t + 3) // 4 * 4 + 4), tail, dtype=torch.float32, device=DEV)
    store[:, :, :t] = x.to(DEV)
    return store[:, :, :t]


def want_layer(x, w, b, d, slope, tanh):
    x = x.double()
    y = torch.nn.Conv1d(w.shape[1], w.shape[0], w.shape[2], dilation=d, padding=(w.shape[2] - 1) // 2 * d,
                        padding_mode="reflect").double()
    with torch.no_grad():
        y.weight.copy_(w.double())
        y.bias.copy_(b.double())
        out = y(F.leaky_relu(x, slope))
    return torch.tanh(out) if tanh else out


def run_layer(conv, x, slope, tanh):
    with _lib.dispatch_log() as log:
        y = conv(x, in_slope=slope, tanh=tanh)
    return y, log.names


@pytest.mark.parametrize("name", list(LAYERS))
def test_reflect_layer_matches_float64(name):
    conv, w, b, slope, tanh = layer(name)
    d, k = LAYERS[name][3], LAYERS[name][2]
    pad = (k - 1) // 2 * d
    lengths = [4096, 4097, 4098, 4099, pad + 1, 200]    # T % 4 = 0..3, the shortest legal row, one all-edge tile
    for t in lengths:
        x = torch.randn(2, w.shape[1], t, generator=torch.Generator().manual_seed(t))
        got, names = run_layer(conv, padded_view(x, float("nan")), slope, tanh)
        want = want_layer(x, w, b, d, slope, tanh)
        assert torch.isfinite(got).all(), (name, t)                     # nothing past the row was read
        assert rel_rms(got.cpu().double(), want) <= 5e-5, (name, t, rel_rms(got.cpu().double(), want))
        zero_tail, names0 = run_layer(conv, padded_view(x, 0.0), slope, tanh)
        assert torch.equal(got, zero_tail) and names == names0, (name, t)
        if t == 4096:
            assert names == [LAYERS[name][6]], (name, names)


def test_reflect_layer_many_tiles_per_cta():
    conv, w, b, slope, tanh = layer("res192_d3")
    t = 24576                                        # 8 rows x 2 row tiles x 96 column tiles: > 10 tiles per CTA
    x = torch.randn(8, 192, t, generator=torch.Generator().manual_seed(7))
    got, names = run_layer(conv, padded_view(x, float("nan")), slope, tanh)
    assert names == ["tc3"]
    assert rel_rms(got.cpu().double(), want_layer(x, w, b, 3, slope, tanh)) <= 5e-5


def test_reflect_layer_bf16_matches_rounded_operands():
    conv, w, b, slope, tanh = layer("res192_d3", precision="bf16")
    x = torch.randn(2, 192, 1027, generator=torch.Generator().manual_seed(3))
    got, names = run_layer(conv, padded_view(x, float("nan")), slope, tanh)
    assert names == ["tc16"]
    want = lowp_conv1d(F.pad(x, (3, 3), mode="reflect"), w, b, precision="bf16", in_slope=slope, dilation=3)
    assert rel_rms(got.cpu().double(), want) <= 1e-5


def test_reflect_needs_pad_plus_one_columns():
    conv, *_ = layer("res64_d27")
    with pytest.raises(RuntimeError, match="reflection padding"):
        conv(torch.randn(1, 64, 27, device=DEV), in_slope=0.2)


# ----------------------------------------------------------------------------- PQMF
def test_pqmf_synthesis_matches_oracle_and_peak():
    pq = PQMF()
    x = torch.randn(3, 4, 5003, generator=torch.Generator().manual_seed(4)) * 0.3
    want = MO.pqmf_synthesis(pq.G.double(), x.double())
    peak = torch.zeros(1, dtype=torch.int32, device=DEV)
    got = pq.synthesis(x.to(DEV), peak=peak)
    assert got.shape == want.shape and rel_rms(got.cpu().double(), want) <= 1e-6
    assert int(peak.item()) == int(got.abs().max().view(torch.int32).item())


def test_pqmf_synthesis_odd_taps():
    pq = PQMF(taps=61)
    x = torch.randn(2, 4, 777, generator=torch.Generator().manual_seed(5)) * 0.3
    want = MO.pqmf_synthesis(pq.G.double(), x.double())
    got = pq.synthesis(x.to(DEV))
    assert got.shape == want.shape == (2, 1, 4 * 777 - 1) and rel_rms(got.cpu().double(), want) <= 1e-6


# ----------------------------------------------------------------------------- generators
GEN_T = {"melgan": 16, "fullband": 20, "multiband": 16, "multiband_zoo": 16, "multiband_short": 4, "fullband_short": 4,
         "odd_factor": 37, "multiband_narrow": 16}


def gpu_model(cls_model, sd):
    cls_model.load_state_dict(sd)
    return cls_model.eval().to(DEV)


def check_wave(got, want):
    assert got.shape == want.shape
    assert rms(got, want) <= 1e-4 and rel_rms(got, want) <= 1e-4, (rms(got, want), rel_rms(got, want))


@pytest.mark.parametrize("case", list(CASES))
def test_generator_matches_oracle(case):
    cls, over, model, sd, _ = build_case(case)
    c = torch.randn(2, model._cfg["in_channels"], GEN_T[case], generator=torch.Generator().manual_seed(2))
    kw = oracle_kwargs(model)
    pqmf = cls == "MultibandMelganGenerator"
    m = gpu_model(model, sd)
    check_wave(m(c.to(DEV)).cpu(), MO.generator(sd, c, **kw))                     # the band signals for multi-band
    check_wave(m.inference(c.to(DEV)).cpu(), MO.inference(sd, c, pqmf=pqmf, **kw))


@pytest.mark.parametrize("case", ["multiband_zoo", "fullband_zoo"])
def test_generator_bench_scale(case):
    from tts_b200 import melgan as M
    if case == "fullband_zoo":   # FullbandMelganConfig: melgan_generator, (8, 8, 2, 2), 4 residual blocks
        model = M.MelganGenerator(num_res_blocks=4)
    else:
        model = M.MultibandMelganGenerator(upsample_factors=(8, 4, 2), num_res_blocks=4)
    from test_melgan_oracle_cpu import melgan_state
    sd = melgan_state(model, 8)
    c = torch.randn(8, 80, 300, generator=torch.Generator().manual_seed(6))
    kw = oracle_kwargs(model)
    pqmf = case == "multiband_zoo"
    want = MO.inference({k: v.to(DEV).double() for k, v in sd.items()}, c.to(DEV).double(), pqmf=pqmf, **kw)
    got = gpu_model(model, sd).inference(c.to(DEV))
    check_wave(got.double(), want)


def test_repeat_poisoned_workspace_and_dispatch():
    model = MultibandMelganGenerator(upsample_factors=(8, 4, 2), num_res_blocks=4)
    from test_melgan_oracle_cpu import melgan_state
    m = gpu_model(model, melgan_state(model, 12))
    c = torch.randn(4, 80, 200, generator=torch.Generator().manual_seed(9)).to(DEV)
    with _lib.dispatch_log() as log:
        a = m.inference(c)
    b = m.inference(c)
    for buf in _lib._workspaces.values():
        buf.view(torch.float32)[: buf.numel() // 4].fill_(float("nan"))
    cc = m.inference(c)
    assert torch.equal(a, b) and torch.equal(a, cc) and torch.isfinite(a).all()
    # conv_pre, then per stage the upsampler and (dilated conv, shortcut, 1x1) per block, all 3xTF32; conv_post (4 rows) FMA
    assert log.names == ["tc3"] + (["tc3"] + ["tc3"] * 3 * 4) * 3 + ["fma"], log.names
    peak = torch.zeros(1, dtype=torch.int32, device=DEV)
    d = m.inference(c, peak=peak)
    assert torch.equal(a, d) and int(peak.item()) == int(a.abs().max().view(torch.int32).item())


def test_glow_tts_to_multiband_melgan_chain():
    """GlowTTS -> vocoder_input(padding=2, [B, T, C] input) -> GAN(MultibandMelganConfig()).inference, against the
    oracle chain."""
    from tts_b200.glow_tts import GlowTTS
    from tts_b200.vocoder import GAN, AudioNorm, MultibandMelganConfig, vocoder_input
    from test_melgan_oracle_cpu import melgan_state
    cfg, sd, x, lens, extra, noise = run_case("default")
    want_mel = GO.inference(sd, x, lens, cfg)["model_outputs"]
    gan = GAN(MultibandMelganConfig()).eval()
    gsd = melgan_state(gan.model_g, 13)
    gan.model_g.load_state_dict(gsd)
    want = MO.inference(gsd, want_mel.transpose(1, 2), pqmf=True, **oracle_kwargs(gan.model_g))
    gan.to(DEV)
    glow = GlowTTS(cfg).eval()
    glow.load_state_dict(sd)
    mel = glow.to(DEV).inference(x.to(DEV), {"x_lengths": lens.to(DEV)})["model_outputs"]
    voc_in = vocoder_input(mel, AudioNorm.identity(), AudioNorm.identity(), padding=2, time_last=False)
    got = gan.model_g.forward(voc_in)
    got = gan.model_g.pqmf_synthesis(got).cpu()
    check_wave(got, want)
    check_wave(gan.inference(mel.transpose(1, 2)).cpu(), want)


@pytest.mark.parametrize("frames, over", [(3, dict(upsample_factors=(8, 4, 2), num_res_blocks=4)),   # conv_pre: T >= 4
                                          (4, dict())])     # (2, 8, 2, 2), 3 blocks: stage 0 has 8 < 10 columns
def test_too_short_input_raises_before_any_launch(frames, over):
    """A reflect pad wider than its layer's input: RuntimeError naming the pad, nothing launched, the output untouched."""
    import ctypes
    from test_melgan_oracle_cpu import melgan_state
    model = MultibandMelganGenerator(**over)
    m = gpu_model(model, melgan_state(model, 2))
    c = torch.randn(2, 80, frames, device=DEV)
    with pytest.raises(RuntimeError, match="reflect-pads"):
        m(c)
    L = _lib.lib()
    h = m._ensure_handle(c.device)
    tout = L.b200tts_melgan_out_len(h, frames)
    out = torch.full((2, 1, 4 * tout), 7.0, device=DEV)
    ws = torch.zeros(max(1, L.b200tts_melgan_workspace_bytes(h, 2, frames)), dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    rc = L.b200tts_melgan_forward(h, _lib.ptr(c), 2, frames, 1, _lib.ptr(out), None, _lib.ptr(ws),
                                  ctypes.c_size_t(ws.numel()), _lib.stream_ptr(DEV))
    torch.cuda.synchronize()
    assert rc == 1 and b"reflect-pads" in L.b200tts_last_error()
    assert _lib.launch_count() == n0 and bool((out == 7.0).all())
