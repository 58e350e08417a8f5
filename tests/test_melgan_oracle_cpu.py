"""MelGAN generators without a GPU: the CPU restatement (tests/melgan_oracle.py) is pinned ``torch.equal`` to the
unmodified reference generators and PQMF -- live where the reference tree imports, through the results recorded under
tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest tests/test_melgan_oracle_cpu.py`` where the
reference is present) -- and the drop-ins' surface (state-dict layout, PQMF buffers, config defaults, setup_generator name
resolution, checkpoint loading, error behaviour) is checked against it."""
import builtins
import dataclasses
import importlib

import pytest
import torch

import melgan_oracle as MO
import ref_import
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200 import melgan as M
from tts_b200 import vocoder as V

# name -> (class, constructor overrides, frames T); "short" cases use T = 4, the shortest input whose conv_pre reflect pad
# is legal (the zoo's multi-band / plain configs upsample 8x first, so stage 0 has 32 >= 28 columns)
CASES = {
    "melgan": ("MelganGenerator", dict(), 6),
    "fullband": ("FullbandMelganGenerator", dict(), 14),   # (2, 8, 2, 2): stage 0 has 2T >= 28 columns
    "multiband": ("MultibandMelganGenerator", dict(), 6),
    "multiband_zoo": ("MultibandMelganGenerator", dict(upsample_factors=(8, 4, 2), num_res_blocks=4), 6),
    "multiband_short": ("MultibandMelganGenerator", dict(upsample_factors=(8, 4, 2), num_res_blocks=4), 4),
    "fullband_short": ("FullbandMelganGenerator", dict(upsample_factors=(8, 8, 2, 2)), 4),
    "odd_factor": ("MelganGenerator", dict(in_channels=16, base_channels=64, upsample_factors=(3, 2), num_res_blocks=2), 9),
    # last stage narrower than the 4 bands (channels 16, 8, 4, 2): the band signals outgrow every stage tensor
    "multiband_narrow": ("MultibandMelganGenerator", dict(base_channels=32), 6),
}
REF_MODULES = {"MelganGenerator": "TTS.vocoder.models.melgan_generator",
               "MultibandMelganGenerator": "TTS.vocoder.models.multiband_melgan_generator",
               "FullbandMelganGenerator": "TTS.vocoder.models.fullband_melgan_generator"}


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    return {k: getattr(importlib.import_module(v), k) for k, v in REF_MODULES.items()}


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def oracle_kwargs(model):
    c = model._cfg
    return dict(upsample_factors=tuple(c["upsample_factors"]), num_res_blocks=c["num_res_blocks"],
                proj_kernel=c["proj_kernel"], res_kernel=c["res_kernel"])


def melgan_state(model, seed):
    """Seeded weights for a generator's layout; the PQMF buffers keep their (deterministic) values."""
    sd = seeded_state_dict(layout(model.state_dict()), seed)
    for k, v in model.state_dict().items():
        if k.startswith("pqmf_layer."):
            sd[k] = v.clone()
    return sd


def build_case(name):
    cls, over, t = CASES[name]
    model = getattr(M, cls)(**over)
    sd = melgan_state(model, 5)
    c = torch.randn(2, model._cfg["in_channels"], t, generator=torch.Generator().manual_seed(1))
    return cls, over, model, sd, c


@pytest.mark.parametrize("case", list(CASES))
def test_melgan_oracle_equals_reference(R, rec, case):
    cls, over, model, sd, c = build_case(case)
    kw = oracle_kwargs(model)
    pqmf = cls == "MultibandMelganGenerator"
    ref = {}

    def reference():
        if not ref:
            net = R[cls](**over).eval()
            net.load_state_dict(sd)
            with torch.no_grad():
                ref["forward"] = net(c.clone())
                ref["inference"] = net.inference(c.clone())
        return ref

    fwd = MO.generator(sd, c, **kw)
    inf = MO.inference(sd, c, pqmf=pqmf, **kw)
    rec.check("forward", fwd, lambda: reference()["forward"])
    rec.check("inference", inf, lambda: reference()["inference"])
    hop = 1
    for u in kw["upsample_factors"]:
        hop *= u
    assert fwd.shape == (2, model._cfg["out_channels"], c.shape[2] * hop)        # forward: the band signals, no PQMF
    assert inf.shape == ((2, 1, 4 * (c.shape[2] + 4) * hop) if pqmf else (2, 1, (c.shape[2] + 4) * hop))   # not trimmed
    if pqmf:   # inference = PQMF synthesis of the padded input's band signals
        assert torch.equal(inf, MO.pqmf_synthesis(sd["pqmf_layer.G"], MO.generator(sd, torch.nn.functional.pad(
            c, (2, 2), mode="replicate"), **kw)))


def test_pqmf_synthesis_equals_reference(R, rec):
    x = torch.randn(3, 4, 37, generator=torch.Generator().manual_seed(2))
    mine = M.PQMF()
    rec.check("synthesis", MO.pqmf_synthesis(mine.G, x), lambda: R["MultibandMelganGenerator"]().pqmf_synthesis(x))


def test_pqmf_odd_taps_equals_reference(R, rec):
    """An odd tap count: the synthesis filter's taps / 2 padding loses one sample (N * Tb - 1 out)."""
    x = torch.randn(2, 4, 29, generator=torch.Generator().manual_seed(3))
    mine = M.PQMF(taps=61)

    def ref():
        return importlib.import_module("TTS.vocoder.layers.pqmf").PQMF(N=4, taps=61, cutoff=0.15, beta=9.0)

    for k in ("H", "G", "updown_filter"):
        rec.check(k, getattr(mine, k), lambda k=k: getattr(ref(), k))
    got = MO.pqmf_synthesis(mine.G, x)
    assert got.shape == (2, 1, 4 * 29 - 1)
    rec.check("synthesis", got, lambda: ref().synthesis(x))


@pytest.mark.parametrize("cls", list(REF_MODULES))
def test_melgan_state_dict_layout_matches_reference(R, rec, cls):
    want = rec.value("layout", lambda: layout(R[cls]().state_dict()))
    mine = getattr(M, cls)().state_dict()
    got = layout(mine)
    assert [(k, s, d) for k, s, d, _ in got] == [(k, s, d) for k, s, d, _ in want]
    if cls == "MultibandMelganGenerator":
        ref_sd = lambda: R[cls]().state_dict()   # noqa: E731
        for k in ("pqmf_layer.H", "pqmf_layer.G", "pqmf_layer.updown_filter"):
            rec.check(k, mine[k], lambda k=k: ref_sd()[k])


CONFIGS = {"MelganConfig": ("TTS.vocoder.configs.melgan_config", V.MelganConfig),
           "MultibandMelganConfig": ("TTS.vocoder.configs.multiband_melgan_config", V.MultibandMelganConfig),
           "FullbandMelganConfig": ("TTS.vocoder.configs.fullband_melgan_config", V.FullbandMelganConfig)}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_melgan_config_defaults_match_reference(R, rec, name):
    mod, mine_cls = CONFIGS[name]
    mine = {f.name: getattr(mine_cls(), f.name) for f in dataclasses.fields(mine_cls) if f.name != "audio"}

    def ref_fields():
        ref = getattr(importlib.import_module(mod), name)()
        return {k: getattr(ref, k) for k in mine}

    assert mine == rec.value("fields", ref_fields)
    if name == "FullbandMelganConfig":
        assert mine["generator_model"] == "melgan_generator"


def test_setup_generator_name_resolution(R, rec):
    def kinds(setup, configs):
        out = {}
        for key, cfg in configs.items():
            try:
                g = setup(cfg)
                out[key] = (type(g).__name__, [(k, tuple(v.shape)) for k, v in g.state_dict().items()])
            except Exception as e:  # noqa: BLE001 - the exception type is the result
                out[key] = (type(e).__name__, None)
        return out

    def cfgs(mod):
        return {"melgan": mod.MelganConfig(), "multiband": mod.MultibandMelganConfig(),
                "fullband": mod.FullbandMelganConfig(),
                "fullband_generator": mod.FullbandMelganConfig(generator_model="fullband_melgan_generator"),
                "mixed_case": mod.MelganConfig(generator_model="MelGAN_Generator"),
                "hifigan_params": mod.HifiganConfig(generator_model="melgan_generator")}

    def ref_kinds():
        ns = type("C", (), {})
        for cls, mod in (("MelganConfig", "melgan_config"), ("MultibandMelganConfig", "multiband_melgan_config"),
                         ("FullbandMelganConfig", "fullband_melgan_config"), ("HifiganConfig", "hifigan_config")):
            setattr(ns, cls, getattr(importlib.import_module("TTS.vocoder.configs." + mod), cls))
        return kinds(importlib.import_module("TTS.vocoder.models").setup_generator, cfgs(ns))

    want = rec.value("kinds", ref_kinds)
    got = kinds(V.setup_generator, cfgs(V))
    for key, (kind, shapes) in want.items():
        if shapes is None:   # the reference raised: the drop-in raises that type (or a subclass of it)
            assert got[key][1] is None, key
            exc = getattr(V, got[key][0], None) or getattr(builtins, got[key][0])
            assert kind in [c.__name__ for c in exc.__mro__], (key, kind, got[key])
        else:
            assert got[key] == (kind, shapes), key
    assert want["hifigan_params"][0] == "KeyError"
    with pytest.raises(KeyError):
        V.setup_generator(V.HifiganConfig(generator_model="melgan_generator"))
    with pytest.raises(ValueError, match="fullband_melgan_generator"):
        V.setup_generator(V.MelganConfig(generator_model="melgan_fb_generator"))
    for name in ("parallel_wavegan_generator", "univnet_generator", "", "gan", "generator", "melgan", "melgan_gen"):
        with pytest.raises(NotImplementedError):
            V.setup_generator(V.MelganConfig(generator_model=name))
    gan = V.GAN(V.MultibandMelganConfig())
    assert type(gan.model_g).__name__ == "MultibandMelganGenerator"
    assert set(k.split(".")[0] for k in gan.state_dict()) == {"model_g"}


def test_reflect_pad_error_type(R, rec):
    model = M.MultibandMelganGenerator(upsample_factors=(8, 4, 2), num_res_blocks=4)
    sd = melgan_state(model, 3)
    c = torch.randn(1, 80, 3)

    def ref_error():
        net = R["MultibandMelganGenerator"](upsample_factors=(8, 4, 2), num_res_blocks=4)
        try:
            net(c)
        except Exception as e:  # noqa: BLE001
            return type(e).__name__
        return None

    want = rec.value("error", ref_error)
    assert want == "RuntimeError"
    with pytest.raises(RuntimeError):
        MO.generator(sd, c, **oracle_kwargs(model))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU path"):
            model(c)


def test_legacy_weight_norm_checkpoint(tmp_path):
    model = M.FullbandMelganGenerator(in_channels=16, base_channels=64, upsample_factors=(4, 2), num_res_blocks=2)
    sd = melgan_state(model, 9)
    legacy = {}
    for k, v in sd.items():
        k = k.replace(".parametrizations.weight.original0", ".weight_g").replace(".parametrizations.weight.original1",
                                                                                 ".weight_v")
        legacy[k] = v
    assert any(k.endswith(".weight_g") for k in legacy)
    path = tmp_path / "melgan.pth"
    torch.save({"model": legacy}, path)
    fresh = M.FullbandMelganGenerator(in_channels=16, base_channels=64, upsample_factors=(4, 2), num_res_blocks=2)
    fresh.load_checkpoint(None, str(path), eval=False)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, sd[k]), k
    c = torch.randn(1, 16, 7)
    kw = oracle_kwargs(fresh)
    assert torch.equal(MO.generator(legacy, c, **kw), MO.generator(sd, c, **kw))
    fresh.load_checkpoint(None, str(path), eval=True)
    assert not fresh.training
    assert torch.equal(fresh.layers[1].weight, MO.conv_weight(sd, "layers.1"))


def test_strict_loading_needs_pqmf_buffers(tmp_path):
    model = M.MultibandMelganGenerator()
    sd = melgan_state(model, 4)
    sd.pop("pqmf_layer.G")
    with pytest.raises(RuntimeError, match="pqmf_layer.G"):
        M.MultibandMelganGenerator().load_state_dict(sd)
    with pytest.raises(NotImplementedError):
        model.pqmf_analysis(torch.zeros(1, 1, 8))
