"""SpeedySpeech (ForwardTTS with the residual conv-BatchNorm encoder and decoder) without a GPU: the CPU restatement in
tests/speedy_speech_oracle.py is pinned ``torch.equal`` to the unmodified reference ``ForwardTTS(SpeedySpeechConfig)
.inference`` -- live where the reference tree imports, through the results recorded under tests/golden/reference/
elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest tests/test_speedy_speech_oracle_cpu.py`` where the reference is
present) -- and the drop-in's surface (state-dict layout, checkpoint loading, the types it builds) is checked against
it."""
import dataclasses
import math

import pytest
import torch

import speedy_speech_oracle as SO
from test_forward_tts_oracle_cpu import KEYS, R, forward_state, make_config, rec, speaker_manager  # noqa: F401
from tts_b200.forward_tts import (FastPitchConfig, ForwardTTS, ForwardTTSArgs, SpeedySpeech, SpeedySpeechConfig)


def conv_bn_params(kernel_size=4, dilations=(1, 2, 4, 8), num_conv_blocks=2):
    return {"kernel_size": kernel_size, "dilations": list(dilations), "num_conv_blocks": num_conv_blocks,
            "num_res_blocks": len(dilations)}


ENC, DEC = SpeedySpeechConfig().model_args.encoder_params, SpeedySpeechConfig().model_args.decoder_params
SMALL = dict(hidden_channels=32, out_channels=16, encoder_params=ENC, decoder_params=DEC)

# name -> (model_args overrides, config overrides, T, frames per token (None: the tie weights, exactly length_scale
#          frames per token), negative BatchNorm gains, extra inference inputs)
CASES = {
    "defaults": ({}, {}, 21, 3, False, {}),
    "min_tokens": ({}, {}, 13, 3, False, {}),                # 13 tokens: the encoder's widest layer (d 4, k 4) + 1
    "min_frames": ({}, {}, 25, None, False, {}),             # 25 frames: the decoder's widest layer (d 8, k 4) + 1
    "kernel_3": (dict(encoder_params=conv_bn_params(3, [1, 2, 4, 1]), decoder_params=conv_bn_params(3)), {}, 17, 3,
                 False, {}),
    "one_conv": (dict(encoder_params=conv_bn_params(4, [1, 2, 4], 1), decoder_params=conv_bn_params(4, [1, 2, 4, 8, 1], 1)),
                 {}, 16, 4, False, {}),
    "three_convs": (dict(encoder_params=conv_bn_params(4, [1, 2, 1], 3), decoder_params=conv_bn_params(4, [1, 4, 1], 3)),
                    {}, 15, 3, False, {}),
    "negative_gamma": ({}, {}, 18, 3, True, {}),
    "length_scale": (dict(length_scale=1.3), {}, 16, 3, False, {}),
    "speaker_embedding": ({}, dict(use_speaker_embedding=True, num_speakers=5), 15, 3, False,
                          {"speaker_ids": torch.tensor([3])}),
}


def speedy_config(args_over, cfg_over, ns=None):
    return make_config("SpeedySpeechConfig", {**SMALL, **args_over}, cfg_over, ns)


def speedy_state(model, seed, frames, negative_gamma=False):
    """forward_state plus BatchNorm statistics: running_var in [0.5, 1.5), running_mean N(0, 0.1), gains 1 + N(0, 0.05)
    (negated with ``negative_gamma``, so that BatchNorm cannot be folded into the conv)."""
    sd = forward_state(model, seed, frames)
    g = torch.Generator().manual_seed(seed + 7)
    for k in sd:
        bn = ".norm." in k or ".postnet.2." in k
        if bn and k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(sd[k].shape, generator=g)
        elif bn and k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
        elif bn and k.endswith("weight"):
            gain = 1.0 + 0.05 * torch.randn(sd[k].shape, generator=g)
            sd[k] = -gain if negative_gamma else gain
    return sd


def run_case(name, seed=11):
    args_over, cfg_over, t, frames, neg, extra = CASES[name]
    cfg = speedy_config(args_over, cfg_over)
    sd = speedy_state(SpeedySpeech(cfg, speaker_manager=speaker_manager(cfg_over)), seed, frames, neg)
    x = torch.randint(0, 40, (1, t), generator=torch.Generator().manual_seed(seed))
    return cfg, sd, x, dict(extra)


def reference_model(R, args_over, cfg_over, sd):
    model = R.M.ForwardTTS(speedy_config(args_over, cfg_over, R), speaker_manager=speaker_manager(cfg_over)).eval()
    model.load_state_dict(sd)
    return model


@pytest.mark.parametrize("case", list(CASES))
def test_speedy_speech_oracle_equals_reference(R, rec, case):  # noqa: F811
    cfg, sd, x, extra = run_case(case)
    got = SO.inference_one(sd, x, cfg.model_args, **extra)
    ref = {}

    def reference():
        if not ref:
            model = reference_model(R, *CASES[case][:2], sd)
            aux = {"d_vectors": extra.get("d_vectors"), "speaker_ids": extra.get("speaker_ids")}
            ref.update(model.inference(x.clone(), aux_input=aux))
        return ref

    for k in KEYS:
        if got[k] is None:
            assert rec.value(k + "_is_none", lambda k=k: reference()[k] is None), k
        else:
            rec.check(k, got[k], lambda k=k: reference()[k])
    if case == "min_tokens":
        assert x.shape[1] == 13
    if case == "min_frames":
        assert int(got["y_lengths"][0]) == 25


@pytest.mark.parametrize("case", ["tokens_12", "frames_24"])
def test_speedy_speech_reference_errors(R, rec, case):  # noqa: F811
    """The reference raises RuntimeError for 12 tokens (encoder) and for 24 frames from 24 tokens (decoder); so does the
    oracle."""
    cfg, sd, x, _ = run_case("min_tokens" if case == "tokens_12" else "min_frames")
    x = x[:, :12] if case == "tokens_12" else x[:, :24]
    with pytest.raises(RuntimeError):
        SO.inference_one(sd, x, cfg.model_args)

    def ref_error():
        model = reference_model(R, {}, {}, sd)
        try:
            model.inference(x.clone(), aux_input={"d_vectors": None, "speaker_ids": None})
        except RuntimeError:
            return "RuntimeError"
        return "none"

    assert rec.value("error", ref_error) == "RuntimeError"


def test_speedy_speech_state_dict_layout_matches_reference(R, rec):  # noqa: F811
    from ref_golden import layout

    def ref_layout():
        args = R.C["SpeedySpeechConfig"].SpeedySpeechConfig().model_args
        args.num_chars = 100
        return layout(R.M.ForwardTTS(R.C["SpeedySpeechConfig"].SpeedySpeechConfig(model_args=args)).state_dict())

    want = rec.value("layout", ref_layout)
    mine = SpeedySpeech(SpeedySpeechConfig(model_args=dataclasses.replace(SpeedySpeechConfig().model_args,
                                                                          num_chars=100))).state_dict()
    got = layout(mine)
    assert len(got) == len(want) == 471
    assert [(k, s, d) for k, s, d, _ in got] == [(k, s, d) for k, s, d, _ in want]


def test_speedy_speech_load_checkpoint_and_init_from_config(tmp_path):
    cfg, sd, _, _ = run_case("defaults")
    m = SpeedySpeech.init_from_config(cfg)
    assert isinstance(m, SpeedySpeech) and m.length_scale == 1.0
    path = tmp_path / "ss.pth"
    torch.save({"model": sd, "step": 5}, path)
    m.load_checkpoint(cfg, str(path), eval=True)
    assert not m.training
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    bad = dict(sd)
    bad.pop("decoder.decoder.postnet.1.bias")
    torch.save({"model": bad}, path)
    with pytest.raises(RuntimeError):
        SpeedySpeech(cfg).load_checkpoint(cfg, str(path))


def test_speedy_speech_builds_residual_conv_bn_only():
    for kind in ("encoder_type", "decoder_type"):
        args = dataclasses.replace(SpeedySpeechConfig().model_args, num_chars=10, **{kind: "fftransformer"})
        with pytest.raises(NotImplementedError, match="residual_conv_bn only"):
            SpeedySpeech(SpeedySpeechConfig(model_args=args))
    with pytest.raises(NotImplementedError, match="residual_conv_bn"):
        SpeedySpeech(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=10)))
    # ForwardTTS still refuses SpeedySpeech's types, and says which class builds them
    with pytest.raises(NotImplementedError, match="SpeedySpeech builds residual_conv_bn"):
        ForwardTTS(SpeedySpeechConfig(model_args=dataclasses.replace(SpeedySpeechConfig().model_args, num_chars=10)))


def test_speedy_speech_oracle_batched_form_equals_per_row_calls():
    cfg, sd, _, _ = run_case("defaults")
    g = torch.Generator().manual_seed(2)
    lens = torch.tensor([21, 13, 17, 14])
    x = torch.randint(0, 40, (4, 21), generator=g)
    out = SO.inference(sd, x, cfg.model_args, x_lengths=lens)
    for i in range(4):
        n = int(lens[i])
        one = SO.inference_one(sd, x[i: i + 1, :n], cfg.model_args)
        m = one["model_outputs"].shape[1]
        assert int(out["y_lengths"][i]) == m
        assert torch.equal(out["model_outputs"][i, :m], one["model_outputs"][0])
        assert float(out["model_outputs"][i, m:].abs().sum()) == 0.0
        assert torch.equal(out["alignments"][i, :m, :n], one["alignments"][0])
        assert torch.equal(out["durations_log"][i, :, :n], one["durations_log"][0])


def round_margin(out, length_scale):
    """The smallest distance of a pre-round duration above 1 from a round-half boundary (format_durations)."""
    w = (torch.exp(out["durations_log"].double()) - 1) * length_scale
    w = w[w >= 1]
    return float((w - w.floor() - 0.5).abs().min()) if w.numel() else math.inf
