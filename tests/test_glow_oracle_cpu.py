"""Glow-TTS without a GPU: the CPU restatement (tests/glow_oracle.py) is pinned ``torch.equal`` to the unmodified
reference ``GlowTTS.inference`` -- live where the reference tree imports, through the results recorded under
tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest tests/test_glow_oracle_cpu.py`` where
the reference is present) -- and the drop-in's surface (state-dict layout, config defaults, checkpoint loading, error
behaviour) is checked against it."""
import contextlib
import dataclasses
import importlib
import math
import sys

import pytest
import torch

import glow_oracle as GO
import ref_import
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200.glow_tts import GlowTTS, GlowTTSConfig

SMALL = dict(hidden_channels_enc=32, hidden_channels_dec=32, hidden_channels_dp=32, out_channels=16,
             num_flow_blocks_dec=3, num_block_layers=2,
             encoder_params={"kernel_size": 3, "dropout_p": 0.1, "num_layers": 2, "num_heads": 2,
                             "hidden_channels_ffn": 64, "input_length": None})

# name -> (config overrides, batch lengths, T, duration-predictor output bias, extra inference inputs)
CASES = {
    "default": (dict(), [17], 17, math.log(3.0), {}),
    "no_prenet": (dict(SMALL, use_encoder_prenet=False), [15], 15, math.log(3.0), {}),
    "mean_only_false": (dict(SMALL, mean_only=False), [15], 15, math.log(3.0), {}),
    "sigmoid_scale": (dict(SMALL, sigmoid_scale=True), [15], 15, math.log(3.0), {}),
    "speaker_embedding": (dict(SMALL, use_speaker_embedding=True, num_speakers=5), [15, 11], 15, math.log(3.0),
                          {"speaker_ids": torch.tensor([3, 1])}),
    "d_vector": (dict(SMALL, use_d_vector_file=True, d_vector_dim=24), [15, 11], 15, math.log(3.0),
                 {"d_vectors": torch.randn(2, 24, generator=torch.Generator().manual_seed(4))}),
    "padded_batch": (dict(SMALL), [21, 13], 21, None, {}),   # quirk 1: the padded tokens get a frame each
    "odd_frames": (dict(SMALL), [21], 21, None, {}),         # quirk 2: 21 frames in, 20 out
    "length_scale": (dict(SMALL, length_scale=1.7), [15, 9], 15, math.log(3.0), {}),
    "noise": (dict(SMALL, inference_noise_scale=0.33), [15, 12], 15, math.log(3.0), {"noise": True}),
}


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    coqpit = sys.modules["coqpit"].Coqpit
    if not hasattr(coqpit, "__iter__"):   # GlowTTS.__init__ iterates its config (glow_tts.py:71)
        coqpit.__iter__ = lambda self: iter([f.name for f in dataclasses.fields(self)])
    return (importlib.import_module("TTS.tts.models.glow_tts"), importlib.import_module("TTS.tts.configs.glow_tts_config"))


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def glow_state(cfg, seed, dp_bias=None):
    """Seeded weights for a GlowTTS config: orthogonal InvConvNear matrices (as the reference initialises them) and,
    with ``dp_bias``, a duration-predictor output bias that gives about exp(dp_bias) - 1 frames per token."""
    sd = seeded_state_dict(layout(GlowTTS(cfg).state_dict()), seed)
    g = torch.Generator().manual_seed(seed + 1)
    for n in range(cfg.num_flow_blocks_dec):
        sd[f"decoder.flows.{3 * n + 1}.weight"] = torch.linalg.qr(torch.randn(cfg.num_splits, cfg.num_splits,
                                                                              generator=g))[0]
    if dp_bias is not None:
        sd["encoder.duration_predictor.proj.bias"] = torch.full((1,), dp_bias)
    return sd


def case_inputs(lengths, t, n_chars, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, n_chars, (len(lengths), t), generator=g)
    return x, torch.tensor(lengths)


@contextlib.contextmanager
def fixed_randn_like(noise):
    """The reference draws torch.randn_like(y_mean) (glow_tts.py:361); substitute a given tensor."""
    orig = torch.randn_like
    torch.randn_like = lambda t, *a, **k: noise.to(t.dtype)
    try:
        yield
    finally:
        torch.randn_like = orig


def _noise_for(sd, x, lens, cfg, extra):
    """The decoder-length noise of a case (the length comes from a noise-free pass of the oracle)."""
    y = GO.inference(sd, x, lens, dataclasses.replace(cfg, inference_noise_scale=0.0), noise=None,
                     **{k: v for k, v in extra.items() if k != "noise"})
    t_dec = y["y_mean"].shape[1]
    return torch.randn(x.shape[0], cfg.out_channels, t_dec, generator=torch.Generator().manual_seed(7))


def run_case(name):
    over, lengths, t, dp_bias, extra = CASES[name]
    cfg = GlowTTSConfig(num_chars=40, **over)
    sd = glow_state(cfg, 11, dp_bias)
    x, lens = case_inputs(lengths, t, 40)
    extra = dict(extra)
    noise = _noise_for(sd, x, lens, cfg, extra) if extra.pop("noise", False) else None
    return cfg, sd, x, lens, extra, noise


KEYS = ("model_outputs", "y_mean", "y_log_scale", "alignments", "durations_log", "total_durations_log")


@pytest.mark.parametrize("case", list(CASES))
def test_glow_oracle_inference_equals_reference(R, rec, case):
    cfg, sd, x, lens, extra, noise = run_case(case)
    got = GO.inference(sd, x, lens, cfg, noise=noise, **extra)
    ref = {}

    def reference():
        if not ref:
            M, C = R
            rcfg = C.GlowTTSConfig(num_chars=40, **CASES[case][0])
            model = M.GlowTTS(rcfg).eval()
            model.load_state_dict(sd)
            aux = {"x_lengths": lens.clone(), "d_vectors": extra.get("d_vectors"), "speaker_ids": extra.get("speaker_ids")}
            with torch.no_grad(), (fixed_randn_like(noise) if noise is not None else contextlib.nullcontext()):
                ref.update(model.inference(x.clone(), aux_input=aux))
        return ref

    for k in KEYS:
        rec.check(k, got[k], lambda k=k: reference()[k])
    assert got["logdet"] is None
    if case == "padded_batch":   # the 13-token row gets one frame per padded token, with no token aligned to them
        y_len = got["y_lengths"]
        assert y_len[1] == y_len[0] == 21
        assert torch.equal(got["y_mean"][1, 13:21], torch.zeros(8, cfg.out_channels))
        assert got["alignments"][1, 13:21].sum() == 0
    if case == "odd_frames":
        assert int(got["y_lengths"][0]) == 21 and got["model_outputs"].shape[1] == 20


@pytest.mark.parametrize("speakers", [False, True])
def test_glow_state_dict_layout_matches_reference(R, rec, speakers):
    over = dict(use_speaker_embedding=True, num_speakers=4) if speakers else {}

    def ref_layout():
        M, C = R
        return layout(M.GlowTTS(C.GlowTTSConfig(num_chars=100, **over)).state_dict())

    want = rec.value("layout", ref_layout)
    got = layout(GlowTTS(GlowTTSConfig(num_chars=100, **over)).state_dict())
    assert [(k, s, d) for k, s, d, _ in got] == [(k, s, d) for k, s, d, _ in want]
    if not speakers:
        assert len(got) == 507 and sum(math.prod(s) for _, s, _, _ in got) == 28604305


def test_glow_config_defaults_match_reference(R, rec):
    mine = dataclasses.asdict(GlowTTSConfig())

    def ref_fields():
        _, C = R
        ref = C.GlowTTSConfig()
        return {k: getattr(ref, k) for k in mine}

    want = rec.value("fields", ref_fields)
    assert mine == want
    assert mine["inference_noise_scale"] == 0.0 and mine["encoder_params"]["input_length"] is None


def test_load_checkpoint_strict_and_eval(tmp_path):
    cfg = GlowTTSConfig(num_chars=40, **SMALL)
    sd = glow_state(cfg, 3)
    path = tmp_path / "glow.pth"
    torch.save({"model": sd, "step": 5}, path)
    m = GlowTTS(cfg)
    m.load_checkpoint(cfg, str(path), eval=False)
    assert m.training
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    m.load_checkpoint(cfg, str(path), eval=True)
    assert not m.training
    inv = m.decoder.flows[1].weight_inv
    assert inv is not None and torch.equal(inv.data, torch.inverse(sd["decoder.flows.1.weight"].float()))
    assert torch.equal(m.decoder.flows[2].wn.in_layers[0].weight,
                       GO.conv_weight(GO.sub(sd, "decoder.flows.2.wn"), "in_layers.0"))
    bad = dict(sd)
    bad.pop("encoder.proj_m.bias")
    torch.save({"model": bad}, path)
    with pytest.raises(RuntimeError):
        GlowTTS(cfg).load_checkpoint(cfg, str(path))


def test_error_behaviour():
    cfg = GlowTTSConfig(num_chars=40, **SMALL)
    m = GlowTTS(cfg)
    x = torch.zeros(1, 5, dtype=torch.int64)
    with pytest.raises(ValueError, match="together"):
        m.inference(x, {"x_lengths": torch.tensor([5]), "d_vectors": torch.ones(1, 8), "speaker_ids": torch.tensor([0])})
    with pytest.raises(ValueError, match="without enabling speaker embedding"):
        m.inference(x, {"x_lengths": torch.tensor([5]), "speaker_ids": torch.tensor([0])})
    for call in (lambda: m(x, torch.tensor([5]), torch.zeros(1, 10, 16)), lambda: m.inference_with_MAS(x),
                 lambda: m.decoder_inference(torch.zeros(1, 10, 16)), m.unlock_act_norm_layers):
        with pytest.raises(NotImplementedError):
            call()
    for enc in ("gated_conv", "residual_conv_bn", "time_depth_separable"):
        with pytest.raises(NotImplementedError):
            GlowTTS(GlowTTSConfig(num_chars=40, encoder_type=enc))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU path"):
            m.inference(x, {"x_lengths": torch.tensor([5])})
