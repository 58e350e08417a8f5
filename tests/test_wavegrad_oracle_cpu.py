"""WaveGrad without a GPU: the CPU restatement (tests/wavegrad_oracle.py) is pinned ``torch.equal`` to the unmodified
reference ``Wavegrad`` -- live where the reference tree imports, through the results recorded under tests/golden/reference/
elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest tests/test_wavegrad_oracle_cpu.py`` where the reference is present)
-- and the drop-in's surface (state-dict layout with and without weight norm, legacy weight-norm keys, the noise
schedules, load_checkpoint, config defaults, setup_model) is checked against it."""
import dataclasses
import importlib

import numpy as np
import pytest
import torch

import ref_import
import wavegrad_oracle as WO
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200 import vocoder as V
from tts_b200 import wavegrad as W

SMALL = dict(in_channels=16, y_conv_channels=8, x_conv_channels=32, dblock_out_channels=[16, 16],
             ublock_out_channels=[32, 16, 16], upsample_factors=[3, 2, 2], upsample_dilations=[[1, 2, 1, 2]] * 3)
# name -> (WavegradArgs overrides, frames T, test-schedule steps or "npy")
CASES = {
    "default": (dict(), 2, 3),
    "weight_norm": (dict(use_weight_norm=True), 2, 3),
    "short_1": (dict(), 1, 3),
    "short_3": (dict(), 3, 2),
    "factor_3": (SMALL, 5, 6),
    "npy_schedule": (SMALL, 4, "npy"),
}


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    return {"model": importlib.import_module("TTS.vocoder.models.wavegrad"),
            "config": importlib.import_module("TTS.vocoder.configs.wavegrad_config"),
            "models": importlib.import_module("TTS.vocoder.models")}


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def npy_beta():
    return np.linspace(2e-6, 2e-2, 5)


def make_config(over, steps):
    cfg = W.WavegradConfig(model_params=W.WavegradArgs(**over))
    if steps != "npy":
        cfg.test_noise_schedule = {"min_val": 1e-6, "max_val": 1e-2, "num_steps": steps}
    return cfg


def ref_config(R, cfg):
    return R["config"].WavegradConfig(model_params=R["model"].WavegradArgs(**dataclasses.asdict(cfg.model_params)),
                                      test_noise_schedule=dict(cfg.test_noise_schedule))


def beta_of(cfg, steps):
    if steps == "npy":
        return npy_beta()
    s = cfg.test_noise_schedule
    return np.linspace(s["min_val"], s["max_val"], s["num_steps"])


def build_case(name):
    over, t, steps = CASES[name]
    cfg = make_config(over, steps)
    model = W.Wavegrad(cfg)
    sd = seeded_state_dict(layout(model.state_dict()), 7)
    g = torch.Generator().manual_seed(3)
    spec = torch.randn(2, cfg.model_params.in_channels, t, generator=g)
    y = torch.randn(2, 1, model.hop_len * t, generator=g)
    ns = torch.rand(2, generator=g)
    return cfg, model, sd, spec, y, ns, steps


@pytest.mark.parametrize("case", list(CASES))
def test_wavegrad_oracle_equals_reference(R, rec, tmp_path, case):
    cfg, model, sd, spec, y, ns, steps = build_case(case)
    args = cfg.model_params
    sched = WO.schedule(beta_of(cfg, steps))
    ref = {}

    def reference():
        if not ref:
            net = R["model"].Wavegrad(ref_config(R, cfg)).eval()
            net.load_state_dict(sd)
            if steps == "npy":
                p = tmp_path / "schedule.npy"
                np.save(p, {"beta": npy_beta()}, allow_pickle=True)
                net.load_noise_schedule(str(p))
            else:
                net.compute_noise_level(beta_of(cfg, steps))
            with torch.no_grad():
                ref["forward"] = net(y.clone(), spec.clone(), ns.clone())
                torch.manual_seed(11)
                ref["inference"] = net.inference(spec.clone())
        return ref

    fwd = WO.forward(sd, y, spec, ns, args)
    torch.manual_seed(11)          # the reference's draw order, replayed
    inf = WO.inference(sd, spec, sched, args)
    rec.check("forward", fwd, lambda: reference()["forward"])
    rec.check("inference", inf, lambda: reference()["inference"])
    assert fwd.shape == y.shape and inf.shape == y.shape
    # supplied noise reproduces the same draws
    torch.manual_seed(11)
    y0 = torch.randn(y.shape)
    zs = torch.stack([torch.randn(y.shape) for _ in range(len(sched["alpha"]) - 1)])   # draw n = N-1 first ...
    zs = torch.flip(zs, [0])                                                             # ... stored at index n - 1
    assert torch.equal(WO.inference(sd, spec, sched, args, init_noise=y0, step_noise=zs), inf)


@pytest.mark.parametrize("steps", [50, 1000, "npy"])
def test_wavegrad_schedule_equals_reference(R, rec, tmp_path, steps):
    cfg = W.WavegradConfig()
    beta = npy_beta() if steps == "npy" else np.linspace(1e-6, 1e-2, steps)
    mine = W.Wavegrad(W.WavegradConfig(model_params=W.WavegradArgs(**SMALL)))
    if steps == "npy":
        p = tmp_path / "schedule.npy"
        np.save(p, {"beta": beta}, allow_pickle=True)
        mine.load_noise_schedule(str(p))
    else:
        mine.compute_noise_level(beta)
    oracle = WO.schedule(beta)
    net = {}

    def ref(k):
        if not net:
            net["m"] = R["model"].Wavegrad(ref_config(R, cfg))
            net["m"].compute_noise_level(beta)
        return getattr(net["m"], k)

    for k in ("beta", "alpha", "alpha_hat", "noise_level", "c1", "c2", "sigma"):
        assert torch.equal(getattr(mine, k), oracle[k]), k
        rec.check(k, oracle[k], lambda k=k: ref(k))
    assert mine.num_steps == len(beta)


@pytest.mark.parametrize("weight_norm", [False, True])
def test_wavegrad_state_dict_layout_matches_reference(R, rec, weight_norm):
    cfg = W.WavegradConfig(model_params=W.WavegradArgs(use_weight_norm=weight_norm))
    mine = [(k, tuple(v.shape)) for k, v in W.Wavegrad(cfg).state_dict().items()]
    want = rec.value("layout", lambda: [(k, tuple(v.shape)) for k, v in
                                        R["model"].Wavegrad(ref_config(R, cfg)).state_dict().items()])
    assert mine == want
    assert any(".parametrizations.weight.original0" in k for k, _ in mine) == weight_norm


def legacy(sd):
    return {k.replace(".parametrizations.weight.original0", ".weight_g").replace(".parametrizations.weight.original1",
                                                                                  ".weight_v"): v for k, v in sd.items()}


def test_wavegrad_legacy_weight_norm_keys_load():
    cfg = W.WavegradConfig(model_params=W.WavegradArgs(**SMALL, use_weight_norm=True))
    model = W.Wavegrad(cfg)
    sd = seeded_state_dict(layout(model.state_dict()), 4)
    old = legacy(sd)
    assert any(k.endswith(".weight_g") for k in old)
    model.load_state_dict(old)
    for name, m in model.named_modules():
        if isinstance(m, torch.nn.Conv1d):
            assert torch.equal(m.weight, WO.conv_weight(old, name)), name
    g = torch.Generator().manual_seed(1)
    spec, y = torch.randn(1, 16, 3, generator=g), torch.randn(1, 1, 36, generator=g)
    assert torch.equal(WO.forward(old, y, spec, torch.tensor([0.5]), cfg.model_params),
                       WO.forward(sd, y, spec, torch.tensor([0.5]), cfg.model_params))


def test_wavegrad_load_checkpoint_eval(tmp_path):
    cfg = W.WavegradConfig(model_params=W.WavegradArgs(**SMALL, use_weight_norm=True))
    model = W.Wavegrad(cfg)
    sd = seeded_state_dict(layout(model.state_dict()), 9)
    path = tmp_path / "model.pth"
    torch.save({"model": sd}, path)
    model.load_checkpoint(cfg, str(path), eval=True)
    assert not model.training
    keys = model.state_dict().keys()
    assert not any("parametrizations" in k for k in keys) and "y_conv.weight" in keys
    assert torch.equal(model.y_conv.weight, WO.conv_weight(sd, "y_conv"))
    assert torch.equal(model.noise_level, WO.schedule(np.linspace(1e-6, 1e-2, 50))["noise_level"])
    train = W.Wavegrad(cfg)
    train.load_checkpoint(cfg, str(path), eval=False)     # the train schedule, weight norm kept
    assert train.num_steps == 1000 and train.training
    assert any("parametrizations" in k for k in train.state_dict())


def test_wavegrad_config_defaults_match_reference(R, rec):
    mine = W.WavegradConfig()
    fields = ["model", "generator_model", "train_noise_schedule", "test_noise_schedule"]
    got = {f: getattr(mine, f) for f in fields}
    got["model_params"] = dataclasses.asdict(mine.model_params)
    want = rec.value("config", lambda: dict({f: getattr(R["config"].WavegradConfig(), f) for f in fields},
                                            model_params={f.name: getattr(R["model"].WavegradArgs(), f.name)
                                                          for f in dataclasses.fields(R["model"].WavegradArgs)}))
    assert got == want
    assert "discriminator_model" not in mine


def test_wavegrad_setup_model_resolution(R, rec):
    want = rec.value("wavegrad_class", lambda: type(R["models"].setup_model(R["config"].WavegradConfig())).__name__)
    assert type(V.setup_model(W.WavegradConfig())).__name__ == want == "Wavegrad"
    assert isinstance(V.setup_model(V.HifiganConfig()), V.GAN)
    gan = dict(model="gan", generator_model="hifigan_generator",       # no discriminator field: resolved by the name
               generator_model_params=V.HifiganConfig().generator_model_params, audio=V.BaseAudioConfig())
    assert isinstance(V.setup_model(gan), V.GAN)
    for cfg in ({"model": "wavernn"}, {}, {"generator_model": "hifigan_generator"}):
        with pytest.raises(NotImplementedError):
            V.setup_model(cfg)


def test_wavegrad_pe_tables_stay_bounded():
    """One set of positional-encoding tables, rebuilt only for a longer input (the reference's cache rule): vocoding
    sentences of many lengths does not accumulate tables."""
    model = W.Wavegrad(W.WavegradConfig(model_params=W.WavegradArgs(**SMALL)))
    cpu = torch.device("cpu")
    longest = 0
    for t in (5, 3, 9, 2, 9, 7, 12, 4):
        ptrs, frames = model._pe_tables(cpu, t)
        longest = max(longest, t)
        assert frames == longest
        tabs = model._pe[2]
        assert [tuple(x.shape) for x in tabs] == [(c, L) for c, L in zip([8, 16, 16], model._film_lengths(longest))]
    # the values of a longer table's first columns are the shorter table's (the kernels read them through the pitch)
    short = W._pe_table(16, model._film_lengths(4)[1])
    assert torch.equal(model._pe[2][1][:, : short.shape[1]], short)


def test_wavegrad_rejects_inconsistent_channels():
    """FiLM i + 1 reads DBlock i's output: a config whose dblock_out_channels differ from reversed(ublock_out_channels)
    cannot run (the reference fails at its first forward); it is refused at construction."""
    with pytest.raises(ValueError):
        W.Wavegrad(W.WavegradConfig(model_params=W.WavegradArgs(**dict(SMALL, dblock_out_channels=[16, 24]))))
