"""ForwardTTS (FastPitch / FastSpeech / FastSpeech2) without a GPU: the CPU restatement (tests/forward_tts_oracle.py) is
pinned ``torch.equal`` to the unmodified reference ``ForwardTTS.inference`` -- live where the reference tree imports,
through the results recorded under tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest
tests/test_forward_tts_oracle_cpu.py`` where the reference is present) -- and the drop-in's surface (state-dict layout,
config defaults, checkpoint loading, error behaviour) is checked against it."""
import dataclasses
import importlib
import math
import types

import pytest
import torch

import forward_tts_oracle as FO
import ref_import
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200.forward_tts import (FastPitchConfig, FastSpeech2Config, FastSpeechConfig, ForwardTTS, ForwardTTSArgs,
                                  SpeedySpeechConfig)

CONFIGS = {"FastPitchConfig": FastPitchConfig, "FastSpeechConfig": FastSpeechConfig,
           "FastSpeech2Config": FastSpeech2Config, "SpeedySpeechConfig": SpeedySpeechConfig}
REF_CONFIGS = {"FastPitchConfig": "fast_pitch_config", "FastSpeechConfig": "fast_speech_config",
               "FastSpeech2Config": "fastspeech2_config", "SpeedySpeechConfig": "speedy_speech_config"}
REF_NAMES = {"FastSpeech2Config": "Fastspeech2Config"}   # the reference's spelling of that class


def ref_config_class(ns, cls_name):
    return getattr(ns.C[cls_name], REF_NAMES.get(cls_name, cls_name))


def _fft(heads=1):
    return {"hidden_channels_ffn": 64, "num_heads": heads, "num_layers": 2, "dropout_p": 0.1}


SMALL = dict(num_chars=40, hidden_channels=32, out_channels=16, duration_predictor_hidden_channels=32,
             pitch_predictor_hidden_channels=32, energy_predictor_hidden_channels=24, encoder_params=_fft(),
             decoder_params=_fft())

# name -> (config class, model_args overrides, config overrides, T, frames per token (None: the tie weights),
#          length_scale, extra inference inputs)
CASES = {
    "fast_pitch": ("FastPitchConfig", {}, {}, 17, 3, None, {}),
    "fast_speech": ("FastSpeechConfig", {}, {}, 15, 3, None, {}),
    "fastspeech2": ("FastSpeech2Config", {}, {}, 15, 3, None, {}),
    "two_heads": ("FastPitchConfig", dict(encoder_params=_fft(2), decoder_params=_fft(2)), {}, 13, 3, None, {}),
    "speaker_embedding": ("FastPitchConfig", {}, dict(use_speaker_embedding=True, num_speakers=5), 14, 3, None,
                          {"speaker_ids": torch.tensor([3])}),
    "d_vector_proj": ("FastPitchConfig", {}, dict(use_d_vector_file=True, d_vector_dim=24), 14, 3, None,
                      {"d_vectors": torch.randn(1, 24, generator=torch.Generator().manual_seed(4))}),
    "d_vector": ("FastPitchConfig", {}, dict(use_d_vector_file=True, d_vector_dim=32), 14, 3, None,
                 {"d_vectors": torch.randn(1, 32, generator=torch.Generator().manual_seed(5))}),
    "length_scale": ("FastPitchConfig", dict(length_scale=1.7), {}, 15, 3, None, {}),
    "ties_2_5": ("FastPitchConfig", dict(length_scale=2.5), {}, 12, None, None, {}),
    "ties_3_5": ("FastPitchConfig", dict(length_scale=3.5), {}, 12, None, None, {}),
}


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    return types.SimpleNamespace(M=importlib.import_module("TTS.tts.models.forward_tts"),
                                 C={k: importlib.import_module(f"TTS.tts.configs.{v}") for k, v in REF_CONFIGS.items()})


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def make_config(cls_name, args_over, cfg_over, ns=None):
    """A config of ``cls_name`` with SMALL (+ overrides) model args; ns: the reference's modules (None: the drop-in's)."""
    base = dict(CONFIGS[cls_name]().model_args.__dict__) if ns is None else None
    if ns is None:
        args = ForwardTTSArgs(**{**base, **SMALL, **args_over})
        return CONFIGS[cls_name](model_args=args, **cfg_over)
    ref_cls = ref_config_class(ns, cls_name)
    defaults = ref_cls().model_args
    kw = {f.name: getattr(defaults, f.name) for f in dataclasses.fields(defaults)}
    args = ns.M.ForwardTTSArgs(**{**kw, **SMALL, **args_over})
    return ref_cls(model_args=args, **cfg_over)


def speaker_manager(cfg_over):
    if cfg_over.get("use_speaker_embedding") or cfg_over.get("use_d_vector_file"):
        return types.SimpleNamespace(num_speakers=cfg_over.get("num_speakers", 0))
    return None


def forward_state(model, seed, frames=None):
    """Seeded weights for a ForwardTTS layout: LayerNorm gains about 1, the real positional-encoding buffer and, with
    ``frames``, a duration-predictor output bias of log(1 + frames) (exactly ``frames`` per token before rounding).
    ``frames=None``: the round-half-even tie weights -- every duration-predictor weight zero and bias ln 2, so
    exp(logw) - 1 is exactly 1 and length_scale alone sets the pre-round value."""
    sd = seeded_state_dict(layout(model.state_dict()), seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in sd:
        if (".norm1." in k or ".norm2." in k) and k.endswith("weight"):
            sd[k] = 1.0 + 0.05 * torch.randn(sd[k].shape, generator=g)
    if "pos_encoder.pe" in sd:
        sd["pos_encoder.pe"] = model.pos_encoder.pe.clone()
    if frames is not None:
        sd["duration_predictor.proj.bias"] = torch.full((1,), math.log(1.0 + frames))
    else:
        for k in list(sd):
            if k.startswith("duration_predictor."):
                sd[k] = torch.zeros_like(sd[k])
        sd["duration_predictor.proj.bias"] = torch.full((1,), math.log(2.0))
    return sd


def run_case(name, seed=11):
    cls_name, args_over, cfg_over, t, frames, _, extra = CASES[name]
    cfg = make_config(cls_name, args_over, cfg_over)
    model = ForwardTTS(cfg, speaker_manager=speaker_manager(cfg_over))
    sd = forward_state(model, seed, frames)
    x = torch.randint(0, 40, (1, t), generator=torch.Generator().manual_seed(seed))
    return cfg, sd, x, dict(extra)


KEYS = ("model_outputs", "alignments", "pitch", "energy", "durations_log")


@pytest.mark.parametrize("case", list(CASES))
def test_forward_tts_oracle_equals_reference(R, rec, case):
    cfg, sd, x, extra = run_case(case)
    got = FO.inference_one(sd, x, cfg.model_args, **extra)
    ref = {}

    def reference():
        if not ref:
            cls_name, args_over, cfg_over = CASES[case][:3]
            model = R.M.ForwardTTS(make_config(cls_name, args_over, cfg_over, R),
                                   speaker_manager=speaker_manager(cfg_over)).eval()
            model.load_state_dict(sd)
            aux = {"d_vectors": extra.get("d_vectors"), "speaker_ids": extra.get("speaker_ids")}
            ref.update(model.inference(x.clone(), aux_input=aux))
        return ref

    for k in KEYS:
        if got[k] is None:
            assert rec.value(k + "_is_none", lambda k=k: reference()[k] is None), k
        else:
            rec.check(k, got[k], lambda k=k: reference()[k])
    if case.startswith("ties"):   # pre-round value exactly 2.5 / 3.5 -> 2 / 4 frames per token (half to even)
        want = 2 if case == "ties_2_5" else 4
        assert torch.equal(got["durations"], torch.full_like(got["durations"], float(want)))
        assert int(got["y_lengths"][0]) == want * x.shape[1]


def test_oracle_batched_form_equals_per_row_calls():
    cfg, sd, _, _ = run_case("fastspeech2")
    g = torch.Generator().manual_seed(2)
    lens = torch.tensor([15, 9, 12, 2])
    x = torch.randint(0, 40, (4, 15), generator=g)
    out = FO.inference(sd, x, cfg.model_args, x_lengths=lens)
    for i in range(4):
        n = int(lens[i])
        one = FO.inference_one(sd, x[i: i + 1, :n], cfg.model_args)
        m = one["model_outputs"].shape[1]
        assert int(out["y_lengths"][i]) == m
        assert torch.equal(out["model_outputs"][i, :m], one["model_outputs"][0])
        assert float(out["model_outputs"][i, m:].abs().sum()) == 0.0
        assert torch.equal(out["alignments"][i, :m, :n], one["alignments"][0])
        for k in ("durations_log", "pitch", "energy"):
            assert torch.equal(out[k][i, :, :n], one[k][0]) and float(out[k][i, :, n:].abs().sum()) == 0.0


@pytest.mark.parametrize("cls_name", ["FastPitchConfig", "FastSpeech2Config"])
def test_forward_tts_state_dict_layout_matches_reference(R, rec, cls_name):
    over = dict(use_speaker_embedding=True, num_speakers=4)

    def ref_layout():
        args = ref_config_class(R, cls_name)().model_args
        args.num_chars = 100
        cfg = ref_config_class(R, cls_name)(model_args=args, **over)
        return layout(R.M.ForwardTTS(cfg, speaker_manager=speaker_manager(over)).state_dict())

    want = rec.value("layout", ref_layout)
    mine = ForwardTTS(CONFIGS[cls_name](model_args=dataclasses.replace(CONFIGS[cls_name]().model_args, num_chars=100),
                                        **over), speaker_manager=speaker_manager(over)).state_dict()
    got = layout(mine)
    assert [(k, s, d) for k, s, d, _ in got] == [(k, s, d) for k, s, d, _ in want]
    assert "pos_encoder.pe" in mine and any(k.startswith("aligner.") for k in mine)
    rec.check("pe", mine["pos_encoder.pe"], lambda: R.M.ForwardTTS(ref_config_class(R, cls_name)(
        model_args=R.M.ForwardTTSArgs(num_chars=100))).state_dict()["pos_encoder.pe"])


@pytest.mark.parametrize("cls_name", list(CONFIGS))
def test_forward_tts_config_defaults_match_reference(R, rec, cls_name):
    mine = dataclasses.asdict(CONFIGS[cls_name]())

    def ref_fields():
        ref = ref_config_class(R, cls_name)()
        out = {k: getattr(ref, k) for k in mine if k != "model_args"}
        out["model_args"] = {f.name: getattr(ref.model_args, f.name) for f in dataclasses.fields(ref.model_args)}
        return out

    assert mine == rec.value("fields", ref_fields)


def test_length_scale_attribute_and_init_multispeaker_rules():
    m = ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10)))
    assert isinstance(m.length_scale, float) and m.length_scale == 1.0
    assert not hasattr(m, "emb_g") and not hasattr(m, "proj_g") and m.embedded_speaker_dim == 0
    with pytest.raises(ValueError, match="SpeakerManager is not provided"):
        ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10), use_speaker_embedding=True))
    sm = types.SimpleNamespace(num_speakers=3)
    m = ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10), use_speaker_embedding=True), speaker_manager=sm)
    assert m.emb_g.weight.shape == (3, 384)
    m = ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10), use_d_vector_file=True, d_vector_dim=512),
                   speaker_manager=sm)
    assert m.proj_g.weight.shape == (384, 512) and m.embedded_speaker_dim == 512 and not hasattr(m, "emb_g")
    m = ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10), use_d_vector_file=True, d_vector_dim=384),
                   speaker_manager=sm)
    assert not hasattr(m, "proj_g")
    m = ForwardTTS.init_from_config(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10, length_scale=1.5)))
    assert m.length_scale == 1.5


def test_load_checkpoint(tmp_path):
    cfg = make_config("FastSpeech2Config", {}, {})
    m = ForwardTTS(cfg)
    sd = forward_state(m, 3, 4)
    path = tmp_path / "fs2.pth"
    torch.save({"model": sd, "step": 5}, path)
    m.load_checkpoint(cfg, str(path), eval=False)
    assert m.training
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    m.load_checkpoint(cfg, str(path), eval=True)
    assert not m.training
    bad = dict(sd)
    bad.pop("decoder.decoder.postnet.bias")
    torch.save({"model": bad}, path)
    with pytest.raises(RuntimeError):
        ForwardTTS(cfg).load_checkpoint(cfg, str(path))


def test_error_behaviour():
    cfg, sd, x, _ = run_case("fast_pitch")
    # one token: the reference's o_en.squeeze() drops the time axis too
    with pytest.raises(RuntimeError):
        FO.inference_one(sd, x[:, :1], cfg.model_args)
    # more frames than the positional encoding holds (5000)
    big = dict(sd)
    big["duration_predictor.proj.bias"] = torch.full((1,), math.log(1.0 + 400))
    with pytest.raises(RuntimeError, match="PositionalEncoding is"):
        FO.inference_one(big, x, cfg.model_args)
    for kind in ("encoder_type", "decoder_type"):
        with pytest.raises(NotImplementedError, match="residual_conv_bn"):
            ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10, **{kind: "residual_conv_bn"})))
    with pytest.raises(NotImplementedError, match="residual_conv_bn"):
        ForwardTTS(SpeedySpeechConfig(model_args=dataclasses.replace(SpeedySpeechConfig().model_args, num_chars=10)))
    m = ForwardTTS(cfg)
    m.load_state_dict(sd)
    with pytest.raises(ValueError, match="together"):
        m.inference(x, {"d_vectors": torch.ones(1, 8), "speaker_ids": torch.tensor([0])})
    with pytest.raises(ValueError, match="without enabling speaker embedding"):
        m.inference(x, {"speaker_ids": torch.tensor([0])})
    with pytest.raises(NotImplementedError):
        m(x, torch.tensor([17]), torch.tensor([40]))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU path"):
            m.inference(x, {})


@pytest.mark.parametrize("case", ["one_token", "too_long"])
def test_forward_tts_reference_errors(R, rec, case):
    """The reference raises RuntimeError for T_en = 1 and for more than 5000 frames."""
    cfg, sd, x, _ = run_case("fast_pitch")
    if case == "one_token":
        x = x[:, :1]
    else:
        sd = dict(sd)
        sd["duration_predictor.proj.bias"] = torch.full((1,), math.log(1.0 + 400))

    def ref_error():
        model = R.M.ForwardTTS(make_config("FastPitchConfig", {}, {}, R)).eval()
        model.load_state_dict(sd)
        try:
            model.inference(x.clone(), aux_input={"d_vectors": None, "speaker_ids": None})
        except RuntimeError:
            return "RuntimeError"
        return "none"

    assert rec.value("error", ref_error) == "RuntimeError"
