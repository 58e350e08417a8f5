"""UnivNet on the GPU: the kernel-prediction GEMM against float64 at every block, each fused LVC layer alone against
float64 (every dilation, hops 8 / 64 / 256 and an odd-factor hop, T = 1, NaN around and past every tensor, no store
outside the output rows), the whole generator against the oracle (tests/univnet_oracle.py, itself pinned to the
reference) on supplied and on seeded noise, batch rows against single-row runs, determinism with a NaN-poisoned
workspace, the pinned dispatch, the split-fp16 range flag and the Tacotron2 -> GAN(UnivnetConfig()) chain."""
import pytest
import torch

import univnet_oracle as UO
from ref_golden import layout, seeded_state_dict
from tts_b200 import _lib
from tts_b200.univnet import UnivnetGenerator

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WAVE_REL_TOL = 1e-4
DEFAULT = dict(in_channels=64, out_channels=1, hidden_channels=32, cond_channels=80, upsample_factors=[8, 8, 4],
               lvc_layers_each_block=4, lvc_kernel_size=3, kpnet_hidden_channels=64, kpnet_conv_size=3, dropout=0.0)


def rel_rms(got, want):
    return float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt().clamp_min(1e-30))


def gpu_model(seed=5, **over):
    p = dict(DEFAULT)
    p.update(over)
    m = UnivnetGenerator(**p).eval()
    sd = seeded_state_dict(layout(m.state_dict()), seed)
    m.load_state_dict(sd)
    return m.to(DEV), sd, p


def sd64(sd):
    return {k: v.to(DEV).double() for k, v in sd.items()}


def want_forward(sd, p, c, noise):
    """The oracle in float64 on the GPU."""
    return UO.generator(sd64(sd), c.to(DEV).double(), noise.to(DEV).double(),
                        upsample_factors=tuple(p["upsample_factors"]), layers=p["lvc_layers_each_block"]).float()


def mel(b, t, ch=80, seed=1):
    return torch.randn(b, ch, t, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("over,t", [(dict(), 7), (dict(), 1), (dict(kpnet_conv_size=5, cond_channels=100), 70),
                                    (dict(lvc_layers_each_block=3, kpnet_hidden_channels=32), 5)])
def test_predict_gemm_against_float64(over, t):
    m, sd, p = gpu_model(**over)
    c = mel(2, t, p["cond_channels"])
    n = p["lvc_layers_each_block"]
    for blk in range(len(p["upsample_factors"])):
        kern, bias = m.predict(blk, c.to(DEV))
        wk, wb = UO.kernel_predictor(sd64(sd), f"lvc_blocks.{blk}.kernel_predictor.", c.to(DEV).double(), layers=n,
                                     hidden=32)
        # wk [B, L, Cin, Cout, K, T] -> [B, T, L, Cout, K, Cin]; wb [B, L, Cout, T] -> [B, T, L, Cout]
        wk = wk.permute(0, 5, 1, 3, 4, 2)
        wb = wb.permute(0, 3, 1, 2)
        assert rel_rms(kern.double(), wk) < 1e-5, (blk, rel_rms(kern.double(), wk))
        assert rel_rms(bias.double(), wb) < 1e-5, (blk, rel_rms(bias.double(), wb))
        # the first and last frame of each row on their own
        for f in (0, t - 1):
            assert rel_rms(kern[:, f].double(), wk[:, f]) < 1e-5


def run_layer(m, blk, layer, x, pred, t, pitch):
    """b200tts_univnet_lvc_layer on x [B, 32, pitch] (NaN past T * hop and after the tensor) -> x_new (NaN-poisoned)."""
    b = x.shape[0]
    x_new = torch.full((b + 1, 32, pitch), float("nan"), device=DEV)
    h = m._ensure_handle(DEV)
    L = _lib.lib()
    with _lib.dispatch_log() as log:
        rc = L.b200tts_univnet_lvc_layer(h, blk, layer, _lib.ptr(x), _lib.ptr(pred), b, t, _lib.ptr(x_new), pitch,
                                         _lib.stream_ptr(DEV))
        torch.cuda.synchronize()
    _lib.check(rc, "univnet_lvc_layer")
    assert log.names == ["univnet_lvc"], log.names
    return x_new


@pytest.mark.parametrize("factors,blk,t", [((8, 8, 4), 0, 3), ((8, 8, 4), 1, 2), ((8, 8, 4), 2, 1), ((8, 8, 4), 2, 3),
                                           ((3, 5, 4), 1, 4), ((3, 5, 4), 0, 5)])
def test_lvc_layer_against_float64(factors, blk, t):
    m, sd, p = gpu_model(upsample_factors=list(factors))
    hop = 1
    for u in factors[:blk + 1]:
        hop *= u
    n = t * hop
    pitch = n + 5
    c = mel(2, t).to(DEV)
    kern, bias = m.predict(blk, c)
    nl = p["lvc_layers_each_block"]
    # pred with NaN after the last frame of the last row
    pred = torch.full((2 * t + 1, nl * (6144 + 64)), float("nan"), device=DEV)
    pred[: 2 * t, : nl * 6144] = kern.reshape(2 * t, -1)
    pred[: 2 * t, nl * 6144:] = bias.reshape(2 * t, -1)
    x = torch.full((3, 32, pitch), float("nan"), device=DEV)
    x[:2, :, :n] = torch.randn(2, 32, n, generator=torch.Generator().manual_seed(3)).to(DEV)
    wk, wb = UO.kernel_predictor(sd64(sd), f"lvc_blocks.{blk}.kernel_predictor.", c.double(), layers=nl, hidden=32)
    for layer in range(nl):          # dilations 1, 3, 9, 27
        got = run_layer(m, blk, layer, x[:2], pred, t, pitch)
        want = UO.lvc_layer(sd64(sd), f"lvc_blocks.{blk}.", layer, x[:2, :, :n].double(), kern.double().permute(
            0, 2, 5, 3, 4, 1)[:, layer], bias.double().permute(0, 2, 3, 1)[:, layer], hop)
        assert torch.isfinite(got[:2, :, :n]).all()
        assert rel_rms(got[:2, :, :n].double() - x[:2, :, :n].double(), want - x[:2, :, :n].double()) < 1e-5, layer
        for f in (0, t - 1):         # first and last frame of each row
            sl = slice(f * hop, (f + 1) * hop)
            assert rel_rms(got[:2, :, sl].double(), want[:, :, sl]) < 1e-5
        assert torch.isnan(got[:, :, n:]).all() and torch.isnan(got[2]).all(), "store outside the output rows"
        # the float64 kernel predictor gives the same layer within the GEMM's error
        want2 = UO.lvc_layer(sd64(sd), f"lvc_blocks.{blk}.", layer, x[:2, :, :n].double(), wk[:, layer], wb[:, layer], hop)
        assert rel_rms(got[:2, :, :n].double(), want2) < 1e-5


@pytest.mark.parametrize("over,t", [(dict(), 1), (dict(), 9), (dict(upsample_factors=[3, 5, 4]), 6),
                                    (dict(lvc_layers_each_block=2, kpnet_conv_size=5, cond_channels=100), 4),
                                    (dict(use_weight_norm=False), 3)])
def test_generator_against_oracle_supplied_noise(over, t):
    m, sd, p = gpu_model(**over)
    c = mel(2, t, p["cond_channels"])
    noise = torch.randn(2, 64, t, generator=torch.Generator().manual_seed(7))
    got = m(c.to(DEV), noise=noise.to(DEV))
    want = want_forward(sd, p, c, noise)
    assert got.shape == want.shape
    assert rel_rms(got, want) <= WAVE_REL_TOL, rel_rms(got, want)


def test_seeded_draws_forward_and_inference():
    m, sd, p = gpu_model()
    c = mel(2, 5)
    torch.manual_seed(21)
    got_f = m(c.to(DEV))
    torch.manual_seed(21)
    want_f = want_forward(sd, p, c, torch.randn(2, 64, 5))
    assert rel_rms(got_f, want_f) <= WAVE_REL_TOL
    torch.manual_seed(22)
    got_i = m.inference(c.to(DEV))
    torch.manual_seed(22)
    torch.randn(2, 64, 5)            # inference's discarded draw
    want_i = want_forward(sd, p, c, torch.randn(2, 64, 5))
    assert rel_rms(got_i, want_i) <= WAVE_REL_TOL
    assert rel_rms(got_i, want_f) > 1e-2   # two draws, not one


def test_batch_rows_equal_single_rows():
    m, sd, p = gpu_model()
    c = mel(32, 6).to(DEV)
    noise = torch.randn(32, 64, 6, generator=torch.Generator().manual_seed(4)).to(DEV)
    full = m(c, noise=noise)
    for b in (0, 1, 17, 31):
        assert torch.equal(full[b:b + 1], m(c[b:b + 1], noise=noise[b:b + 1])), b


def test_repeatable_over_poisoned_workspace():
    m, sd, p = gpu_model()
    c, noise = mel(3, 11).to(DEV), torch.randn(3, 64, 11, generator=torch.Generator().manual_seed(2)).to(DEV)
    a = m(c, noise=noise)
    h = m._ensure_handle(DEV)
    ws = _lib.workspace(DEV, _lib.lib().b200tts_univnet_workspace_bytes(h, 3, 11), "univnet")
    ws.view(torch.uint8).fill_(0xFF)   # NaN bit patterns everywhere
    b = m(c, noise=noise)
    assert torch.equal(a, b)


def test_dispatch_ids():
    m, sd, p = gpu_model()
    c, noise = mel(1, 4).to(DEV), torch.randn(1, 64, 4).to(DEV)
    with _lib.dispatch_log() as log:
        m(c, noise=noise)
        torch.cuda.synchronize()
    names = log.names
    blocks = [i for i, n in enumerate(names) if n == "univnet_predict"]
    assert len(blocks) == 3, names
    assert names.count("univnet_lvc") == 12, names
    for i in blocks:                 # per block: prediction GEMM, the upsampler, then the four LVC layers
        assert names[i + 2: i + 6] == ["univnet_lvc"] * 4, names


def test_fp16_range_flag():
    m, sd, p = gpu_model()
    with torch.no_grad():
        m.lvc_blocks[0].kernel_predictor.kernel_conv.bias.fill_(1e5)   # every predicted kernel of block 0 past 65504
    m.repack()
    c, noise = mel(1, 3).to(DEV), torch.randn(1, 64, 3).to(DEV)
    m(c, noise=noise)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="65504"):
        m(c, noise=noise)
    # the flag is reported once: a model in range runs again
    m2, sd2, p2 = gpu_model()
    assert torch.isfinite(m2(c, noise=noise)).all()


def test_tacotron2_to_univnet_gan():
    """The zoo pairing: Tacotron2-DDC -> vocoder_input -> GAN(UnivnetConfig()) with a reference-format state dict."""
    from test_tacotron2_gpu import make, tokens
    from tts_b200 import vocoder as V

    _, taco, _ = make(max_decoder_steps=20, double_decoder_consistency=True)
    text, lens = tokens([10, 6])
    mel_out = taco.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})["model_outputs"]
    norm = V.AudioNorm(signal_norm=True, symmetric_norm=True, max_norm=4.0, clip_norm=True, min_level_db=-100.0,
                       ref_level_db=20.0)
    voc_in = V.vocoder_input(mel_out, norm, norm, padding=0, time_last=False)
    gan = V.GAN(V.UnivnetConfig())
    sd = seeded_state_dict(layout(gan.state_dict()), 4)
    gan.load_state_dict(sd)
    gan.eval().to(DEV)
    assert type(gan.model_g).__name__ == "UnivnetGenerator"
    noise = torch.randn(voc_in.shape[0], 64, voc_in.shape[2], generator=torch.Generator().manual_seed(6))
    got = gan.model_g(voc_in, noise=noise.to(DEV))
    gsd = {k[len("model_g."):]: v for k, v in sd.items() if k.startswith("model_g.")}
    want = UO.generator(sd64(gsd), voc_in.double(), noise.to(DEV).double()).float()
    assert got.shape == (2, 1, voc_in.shape[2] * 256)
    assert rel_rms(got, want) <= WAVE_REL_TOL, rel_rms(got, want)
    torch.manual_seed(3)
    assert gan.inference(voc_in).shape == got.shape
