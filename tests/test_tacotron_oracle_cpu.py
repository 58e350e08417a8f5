"""Tacotron (1) without a GPU: the CPU restatement (tests/tacotron_oracle.py) is pinned ``torch.equal`` to the
unmodified reference ``Tacotron.inference`` -- live where the reference tree imports, through the results recorded under
tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest tests/test_tacotron_oracle_cpu.py``
where the reference is present) -- and the drop-in's surface (config defaults, state-dict layout, load_checkpoint,
the options it rejects) is checked against it."""
import dataclasses
import importlib
import sys

import pytest
import torch

import ref_import
import tacotron_oracle as TO
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200 import tacotron as TC

# name -> (config overrides, stopnet bias, stopnet gain, token lengths)
CASES = {
    "default": (dict(max_decoder_steps=10), -30.0, 40.0, [9, 4]),
    "ddc": (dict(double_decoder_consistency=True, max_decoder_steps=10), -30.0, 40.0, [9, 4]),
    "softmax": (dict(attention_norm="softmax", max_decoder_steps=10), -30.0, 40.0, [8, 5]),
    "no_location": (dict(location_attn=False, max_decoder_steps=10), -30.0, 40.0, [8, 5]),
    "dca": (dict(attention_type="dynamic_convolution", max_decoder_steps=10), -30.0, 40.0, [8, 5]),
    "prenet_bn": (dict(prenet_type="bn", max_decoder_steps=10), -30.0, 40.0, [8, 5]),
    "dropout_at_inference": (dict(prenet_dropout_at_inference=True, max_decoder_steps=10), -30.0, 40.0, [8, 5]),
    "memory_size_5": (dict(memory_size=5, max_decoder_steps=10), -30.0, 40.0, [8, 5]),
    "memory_size_1": (dict(memory_size=1, max_decoder_steps=10), -30.0, 40.0, [8, 5]),
    "r_below_r_init": (dict(r=3, max_decoder_steps=8), -30.0, 40.0, [7, 3]),
    "out_channels_80": (dict(out_channels=80, max_decoder_steps=8), -30.0, 40.0, [7, 3]),
    "out_channels_513": (dict(out_channels=513, max_decoder_steps=8), -30.0, 40.0, [7, 3]),
    "max_decoder_steps_cut": (dict(max_decoder_steps=5), -30.0, 40.0, [6, 6]),
    "one_token": (dict(max_decoder_steps=6), -30.0, 40.0, [1]),
    "stop_logit_high_at_step_0": (dict(max_decoder_steps=20), 30.0, 40.0, [6, 1, 9]),
    "attention_stop": (dict(attention_type="dynamic_convolution", max_decoder_steps=40), -30.0, 40.0, [5, 6]),
    "rows_stop_at_different_steps": (dict(max_decoder_steps=45), -0.30, -40.0, [12, 7, 1, 10]),
}


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    coqpit = sys.modules["coqpit"].Coqpit
    if not hasattr(coqpit, "__iter__"):   # the model's __init__ iterates its config's fields
        coqpit.__iter__ = lambda self: iter([f.name for f in dataclasses.fields(self)])
    return (importlib.import_module("TTS.tts.models.tacotron").Tacotron,
            importlib.import_module("TTS.tts.configs.tacotron_config").TacotronConfig)


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def build_case(name):
    over, bias, gain, lens = CASES[name]
    cfg = TC.TacotronConfig(num_chars=40, **over)
    model = TC.Tacotron(cfg)
    sd = TO.seeded_weights(seeded_state_dict(layout(model.state_dict()), 13), 17, stop_bias=bias, stop_gain=gain)
    g = torch.Generator().manual_seed(3)
    text = torch.zeros(len(lens), max(lens), dtype=torch.long)
    for b, n in enumerate(lens):
        text[b, :n] = torch.randint(1, 40, (n,), generator=g)
    return cfg, sd, text, torch.tensor(lens)


def case_r(name, cfg):
    return 2 if name == "r_below_r_init" else cfg.r


def ref_config(R, cfg):
    fields = {f.name for f in dataclasses.fields(R[1])}
    return R[1](**{k: v for k, v in dataclasses.asdict(cfg).items() if k in fields})


@pytest.mark.parametrize("case", list(CASES))
def test_tacotron_oracle_equals_reference(R, rec, case):
    cfg, sd, text, lens = build_case(case)
    r = case_r(case, cfg)
    ref = {}

    def reference():
        if not ref:
            net = R[0](ref_config(R, cfg))
            net.load_state_dict(sd)
            net.eval()
            net.decoder.set_r(r)
            torch.manual_seed(29)
            ref["rows"] = [net.inference(text[b:b + 1, :int(lens[b])]) for b in range(len(lens))]
        return ref

    torch.manual_seed(29)
    got = TO.inference(sd, text, lens, cfg, r=r)
    for b in range(len(lens)):
        s, n = got["steps"][b], int(lens[b])
        for k, v in (("model_outputs", got["model_outputs"][b:b + 1, :s * r]),
                     ("decoder_outputs", got["decoder_outputs"][b:b + 1, :s * r]),
                     ("alignments", got["alignments"][b:b + 1, :s, :n]),
                     ("stop_tokens", got["stop_tokens"][b:b + 1, :s])):
            rec.check(f"{k}_{b}", v, lambda b=b, k=k: reference()["rows"][b][k])
    steps, mx = got["steps"], cfg.max_decoder_steps
    stops = [got["stop_tokens"][b, :steps[b], 0] for b in range(len(lens))]
    if case == "max_decoder_steps_cut":
        assert steps == [mx + 1, mx + 1]
    if case == "one_token":   # a one-token row's only weight is 1.0: the attention test stops it after its first step
        assert steps == [1]
    if case == "stop_logit_high_at_step_0":   # the len / 4 gate holds the stop until t > len / 4
        assert all(lg[0] > 0 for lg in got["logits"]) and steps == [2, 1, 3]
    if case == "attention_stop":   # the monotonic attention reaches the last token: stopped by that test alone
        assert all(1 < s <= mx for s in steps) and all(float(st.max()) < 0.6 for st in stops)
    if case == "rows_stop_at_different_steps":
        assert len(set(steps)) > 1 and any(s <= mx for s in steps)


def test_tacotron_supplied_draws_replay_oracle():
    """Supplying the prenet dropout masks reproduces the oracle's own-draw run bit for bit: seeded, the own-draw path
    takes F.dropout on [1, 256] and [1, 128] per step; drawing the same masks (bernoulli(0.5) in the same order) and
    passing them as ``draws["dropout"]`` keeps and doubles the same units."""
    cfg, sd, text, lens = build_case("dropout_at_inference")
    torch.manual_seed(1)
    own = TO.inference(sd, text, lens, cfg)
    torch.manual_seed(1)
    drop = torch.zeros(len(lens), cfg.max_decoder_steps + 1, 2, 256, dtype=torch.bool)
    for b in range(len(lens)):
        for t in range(own["steps"][b]):
            drop[b, t, 0] = torch.empty(1, 256).bernoulli_(0.5)[0].bool()
            drop[b, t, 1, :128] = torch.empty(1, 128).bernoulli_(0.5)[0].bool()
    sup = TO.inference(sd, text, lens, cfg, draws={"dropout": drop})
    for k in ("model_outputs", "alignments", "stop_tokens"):
        assert torch.equal(own[k], sup[k]), k


def test_tacotron_config_defaults_match_reference(R, rec):
    cfg = TC.TacotronConfig()
    for f in dataclasses.fields(cfg):
        want = rec.value(f.name, lambda f=f: getattr(R[1](), f.name))
        assert getattr(cfg, f.name) == want, f.name


@pytest.mark.parametrize("over", [dict(), dict(double_decoder_consistency=True),
                                  dict(attention_type="dynamic_convolution", prenet_type="bn"), dict(memory_size=5),
                                  dict(decoder_output_dim=128, out_channels=80)],
                         ids=["default", "ddc", "dca_bn", "memory_size", "no_pre_highway"])
def test_tacotron_state_dict_layout_matches_reference(R, rec, over):
    got = [(k, s, d) for k, s, d, _ in layout(TC.Tacotron(TC.TacotronConfig(num_chars=40, **over)).state_dict())]
    want = rec.value("layout", lambda: [(k, s, d) for k, s, d, _ in
                                        layout(R[0](R[1](num_chars=40, **over)).state_dict())])
    assert got == [tuple(x) for x in want]


@pytest.mark.parametrize("where", ["state", "config", "new_config"])
def test_tacotron_load_checkpoint_r(R, rec, tmp_path, where):
    cfg, sd, text, lens = build_case("r_below_r_init")
    state = {"model": sd}
    if where == "state":
        state["r"] = 1
    elif where == "config":
        state["config"] = {"r": 2}
    path = tmp_path / "ckpt.pth"
    torch.save(state, path)
    new_cfg = TC.TacotronConfig(num_chars=40, r=3)
    model = TC.Tacotron(cfg)
    model.load_checkpoint(new_cfg, str(path), eval=True)
    assert not model.training

    def reference():
        net = R[0](ref_config(R, cfg))
        net.load_checkpoint(ref_config(R, new_cfg), str(path), eval=True)
        return net.decoder.r

    assert model.decoder.r == rec.value("r", reference)
    assert torch.equal(model.state_dict()["last_linear.bias"], sd["last_linear.bias"])


@pytest.mark.parametrize("over", [dict(attention_type="graves"), dict(attention_win=True), dict(windowing=True),
                                  dict(use_forward_attn=True), dict(forward_attn_mask=True),
                                  dict(transition_agent=True), dict(use_gst=True), dict(use_capacitron_vae=True),
                                  dict(num_speakers=4), dict(use_speaker_embedding=True), dict(use_d_vector_file=True),
                                  dict(bidirectional_decoder=True), dict(encoder_in_features=512),
                                  dict(decoder_in_features=512), dict(model="tacotron2")],
                         ids=lambda d: "_".join(f"{k}={v}" for k, v in d.items()))
def test_tacotron_out_of_scope_options_raise(over):
    with pytest.raises(NotImplementedError):
        TC.Tacotron(TC.TacotronConfig(num_chars=40, **over))


def test_tacotron_forward_and_training_mode_inference_raise():
    model = TC.Tacotron(TC.TacotronConfig(num_chars=40))
    with pytest.raises(NotImplementedError):
        model.forward(None, None)
    with pytest.raises(NotImplementedError):   # training mode: the encoder prenet's dropout would be active
        model.train().inference(torch.ones(1, 3, dtype=torch.long))


def test_tacotron2_still_rejects_tacotron_model():
    from tts_b200 import tacotron2 as T2
    with pytest.raises(NotImplementedError, match="tts_b200.tacotron.Tacotron"):
        T2.Tacotron2(T2.Tacotron2Config(num_chars=40, model="tacotron"))
