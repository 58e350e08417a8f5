"""Overflow / Neural-HMM without a GPU: the CPU restatement (tests/overflow_oracle.py) is pinned ``torch.equal`` to the
unmodified reference ``Overflow`` / ``NeuralhmmTTS`` -- live where the reference tree imports, through the results
recorded under tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest
tests/test_overflow_oracle_cpu.py`` where the reference is present) -- and the drop-in's surface (config defaults,
state-dict layout, load_checkpoint) is checked against it."""
import dataclasses
import importlib
import sys

import pytest
import torch

import overflow_oracle as OO
import ref_import
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200 import overflow as OV

SMALL = dict(encoder_in_out_features=64, prenet_dim=32, memory_rnn_dim=64, outputnet_size=[64])
SMALL_DEC = dict(SMALL, hidden_channels_dec=24, num_flow_blocks_dec=3, num_block_layers=2)
# name -> (model, config overrides, aux_input overrides, token lengths, reference draws its own noise)
CASES = {
    "overflow_default": ("overflow", dict(sampling_temp=0.0), {}, [9, 6], False),
    "neuralhmm_default": ("neuralhmm", dict(prenet_dropout_at_inference=False), {}, [9, 6], False),
    "overflow_sampled": ("overflow", SMALL_DEC, dict(sampling_temp=0.334), [8, 5], True),
    "neuralhmm_sampled": ("neuralhmm", dict(SMALL, sampling_temp=0.2), {}, [8, 5], True),
    "max_sampling_time": ("overflow", dict(SMALL_DEC, sampling_temp=0.0), dict(max_sampling_time=23), [12, 4], False),
    "spp_1": ("neuralhmm", dict(SMALL, state_per_phone=1, prenet_dropout_at_inference=False), {}, [7, 3], False),
    "spp_3": ("overflow", dict(SMALL_DEC, state_per_phone=3, sampling_temp=0.0), {}, [5, 4], False),
    "ar_order_2": ("neuralhmm", dict(SMALL, ar_order=2, prenet_dropout_at_inference=False), {}, [6, 6], False),
    "two_outputnet_layers": ("overflow", dict(SMALL_DEC, outputnet_size=[64, 48], sampling_temp=0.0), {}, [6, 5],
                             False),
    "per_channel_mean_std": ("overflow", dict(SMALL_DEC, sampling_temp=0.0), {}, [6, 5], False),
}


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    coqpit = sys.modules["coqpit"].Coqpit
    if not hasattr(coqpit, "__iter__"):   # Overflow.__init__ iterates its config's fields
        coqpit.__iter__ = lambda self: iter([f.name for f in dataclasses.fields(self)])
    return {"overflow": (importlib.import_module("TTS.tts.models.overflow").Overflow,
                         importlib.import_module("TTS.tts.configs.overflow_config").OverflowConfig),
            "neuralhmm": (importlib.import_module("TTS.tts.models.neuralhmm_tts").NeuralhmmTTS,
                          importlib.import_module("TTS.tts.configs.neuralhmm_tts_config").NeuralhmmTTSConfig)}


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def drop_in(kind):
    return (OV.Overflow, OV.OverflowConfig) if kind == "overflow" else (OV.NeuralhmmTTS, OV.NeuralhmmTTSConfig)


def build_case(name):
    kind, over, aux, lens, _ = CASES[name]
    model_cls, cfg_cls = drop_in(kind)
    cfg = cfg_cls(num_chars=40, **over)
    model = model_cls(cfg)
    if name == "per_channel_mean_std":
        g = torch.Generator().manual_seed(5)
        model.update_mean_std({"mean": (torch.randn(80, generator=g) * 0.5).tolist(),
                               "std": (1.0 + torch.rand(80, generator=g)).tolist()})
    sd = OO.seeded_weights(seeded_state_dict(layout(model.state_dict()), 13), 17)
    g = torch.Generator().manual_seed(3)
    text = torch.zeros(len(lens), max(lens), dtype=torch.long)
    for b, n in enumerate(lens):
        text[b, :n] = torch.randint(1, 40, (n,), generator=g)
    return kind, cfg, sd, text, torch.tensor(lens), aux


def ref_config(R, kind, cfg):
    fields = {f.name for f in dataclasses.fields(R[kind][1])}
    return R[kind][1](**{k: v for k, v in dataclasses.asdict(cfg).items() if k in fields})


@pytest.mark.parametrize("case", list(CASES))
def test_overflow_oracle_equals_reference(R, rec, case):
    kind, cfg, sd, text, lens, aux = build_case(case)
    ref = {}

    def reference():
        if not ref:
            net = R[kind][0](ref_config(R, kind, cfg))
            if sd["mean"].dim():   # per-channel statistics: the buffers take their shape from update_mean_std
                net.update_mean_std({"mean": sd["mean"].tolist(), "std": sd["std"].tolist()})
            net.load_state_dict(sd)
            net.eval()
            torch.manual_seed(29)
            ref["rows"] = [net.inference(text[b:b + 1, :int(lens[b])], aux_input=dict(aux)) for b in range(len(lens))]
        return ref

    torch.manual_seed(29)
    got = OO.inference(sd, text, lens, cfg, has_decoder=kind == "overflow", temp=aux.get("sampling_temp"),
                       max_t=aux.get("max_sampling_time"))
    for b in range(len(lens)):
        n = int(got["hmm_outputs_len"][b])
        rec.check(f"hmm_outputs_{b}", got["hmm_outputs"][b:b + 1, :n], lambda b=b: reference()["rows"][b]["hmm_outputs"])
        rec.check(f"hmm_outputs_len_{b}", got["hmm_outputs_len"][b:b + 1],
                  lambda b=b: reference()["rows"][b]["hmm_outputs_len"])
        a = got["alignments"][b:b + 1, :n + 1]
        w = int(a.sum(dim=(0, 1)).nonzero().max()) + 1
        rec.check(f"alignments_{b}", a[:, :, :w], lambda b=b: reference()["rows"][b]["alignments"])
        m = int(got["model_outputs_len"][b])
        mo = got["model_outputs"][b:b + 1, :m] if kind == "overflow" else got["model_outputs"][b:b + 1, :n]
        rec.check(f"model_outputs_{b}", mo, lambda b=b: reference()["rows"][b]["model_outputs"])
        rec.check(f"model_outputs_len_{b}", got["model_outputs_len"][b:b + 1],
                  lambda b=b: reference()["rows"][b]["model_outputs_len"])
    assert all(mg > 0 for mg in got["margins"])
    # the seeded weights give each row states of different lengths, so the duration path is exercised per state
    for b in range(len(lens)):
        assert len(set(OO.state_durations(got["alignments"][b], int(got["hmm_outputs_len"][b])))) > 1, b
    if case == "max_sampling_time":
        assert int(got["hmm_outputs_len"][0]) == 23


def test_overflow_supplied_draws_replay_oracle():
    """Supplying the draws reproduces the oracle's own-draw run bit for bit: seeded, the own-draw path takes one
    Normal(mean, std * temp).sample() of [1, 1, C] per frame and row; drawing the same standard normals
    (torch.normal(0, 1) on [1, 1, C], in the same order) and passing them as ``draws["noise"]`` gives mean + (std * temp)
    * noise, the same numbers."""
    kind, cfg, sd, text, lens, aux = build_case("overflow_sampled")
    torch.manual_seed(1)
    own = OO.inference(sd, text, lens, cfg, has_decoder=True, temp=0.334)
    torch.manual_seed(1)
    noise = torch.zeros(len(lens), cfg.max_sampling_time, 80)
    for b in range(len(lens)):
        for t in range(int(own["hmm_outputs_len"][b])):
            noise[b, t] = torch.normal(torch.zeros(1, 1, 80), torch.ones(1, 1, 80)).flatten()
    sup = OO.inference(sd, text, lens, cfg, has_decoder=True, temp=0.334, draws={"noise": noise})
    for k in ("hmm_outputs", "hmm_outputs_len", "alignments", "model_outputs"):
        assert torch.equal(own[k], sup[k]), k
    c = OO.inference(sd, text, lens, cfg, has_decoder=True, temp=0.0)
    assert not torch.equal(own["hmm_outputs"][0, :5], c["hmm_outputs"][0, :5])


@pytest.mark.parametrize("kind", ["overflow", "neuralhmm"])
def test_overflow_config_defaults_match_reference(R, rec, kind):
    cfg = drop_in(kind)[1]()
    for f in dataclasses.fields(cfg):
        want = rec.value(f.name, lambda f=f: getattr(R[kind][1](), f.name))
        assert getattr(cfg, f.name) == want, f.name
    if kind == "overflow":
        assert cfg.sampling_temp == 0.334 and cfg.prenet_dropout_at_inference is False
    else:
        assert cfg.sampling_temp == 0 and cfg.prenet_dropout_at_inference is True


@pytest.mark.parametrize("kind", ["overflow", "neuralhmm"])
def test_overflow_state_dict_layout_matches_reference(R, rec, kind):
    model_cls, cfg_cls = drop_in(kind)
    model = model_cls(cfg_cls(num_chars=40))
    got = [(k, s, d) for k, s, d, _ in layout(model.state_dict())]
    want = rec.value("layout", lambda: [(k, s, d) for k, s, d, _ in
                                        layout(R[kind][0](R[kind][1](num_chars=40)).state_dict())])
    assert got == [tuple(x) for x in want]
    assert len(got) == (427 if kind == "overflow" else 43)
    n = sum(p.numel() for p in model.parameters())
    assert round(n / 1e6, 1) == (28.4 if kind == "overflow" else 15.2)


def test_overflow_load_checkpoint_matches_reference(R, rec, tmp_path):
    kind, cfg, sd, text, lens, aux = build_case("per_channel_mean_std")
    path = tmp_path / "ckpt.pth"
    torch.save({"model": sd}, path)
    model = OV.Overflow(cfg)
    model.load_checkpoint(cfg, str(path), eval=True)
    assert not model.training and model.mean.shape == (80,)
    got = model.state_dict()

    def reference():
        net = R[kind][0](ref_config(R, kind, cfg))
        net.update_mean_std({"mean": torch.zeros(80).tolist(), "std": torch.ones(80).tolist()})
        net.load_checkpoint(ref_config(R, kind, cfg), str(path), eval=True)
        return net.state_dict()

    want_keys = rec.value("keys", lambda: list(reference().keys()))
    assert list(got.keys()) == want_keys
    rec.check("weight_inv_0", got["decoder.glow_decoder.flows.1.weight_inv"],
              lambda: reference()["decoder.glow_decoder.flows.1.weight_inv"])
