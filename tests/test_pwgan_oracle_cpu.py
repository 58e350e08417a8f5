"""Parallel WaveGAN without a GPU: the CPU restatement (tests/pwgan_oracle.py) is pinned ``torch.equal`` to the unmodified
reference generator on the reference's own seeded noise draw -- live where the reference tree imports, through the results
recorded under tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest
tests/test_pwgan_oracle_cpu.py`` where the reference is present) -- and the drop-in's surface (config defaults, state-dict
layout, setup_generator / GAN, legacy weight-norm checkpoints, error behaviour) is checked against it."""
import dataclasses
import importlib

import pytest
import torch

import pwgan_oracle as PO
import ref_import
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200 import vocoder as V
from tts_b200.pwgan import ParallelWaveganGenerator

REF_MODULE = "TTS.vocoder.models.parallel_wavegan_generator"

# name -> (constructor overrides, frames T)
CASES = {
    "default_T1": (dict(), 1),
    "default_T3": (dict(), 3),
    "default_T40": (dict(), 40),
    "factors_3_5_4": (dict(upsample_factors=[3, 5, 4]), 6),
    "stacks_2_blocks_20": (dict(stacks=2, num_res_blocks=20), 4),
    "no_weight_norm": (dict(use_weight_norm=False), 3),
}


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    return importlib.import_module(REF_MODULE).ParallelWaveganGenerator


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def oracle_kwargs(m):
    return dict(upsample_factors=tuple(m.upsample_factors), num_res_blocks=m.num_res_blocks, stacks=m.stacks)


@pytest.mark.parametrize("case", list(CASES))
def test_pwgan_oracle_equals_reference(R, rec, case):
    over, t = CASES[case]
    mine = ParallelWaveganGenerator(**over)
    sd = seeded_state_dict(layout(mine.state_dict()), 5)
    c = torch.randn(2, 80, t, generator=torch.Generator().manual_seed(1))
    hop = mine.upsample_scale
    ref = {}

    def reference():
        if not ref:
            net = R(**over).eval()
            net.load_state_dict(sd)
            with torch.no_grad():
                torch.manual_seed(21)
                ref["forward"] = net(c.clone())
                torch.manual_seed(22)
                ref["inference"] = net.inference(c.clone())
        return ref

    torch.manual_seed(21)                      # the reference's draw: torch.randn([B, 1, T * hop]) on the CPU generator
    fwd = PO.generator(sd, c, torch.randn([2, 1, t * hop]), **oracle_kwargs(mine))
    torch.manual_seed(22)
    inf = PO.inference(sd, c, torch.randn([2, 1, (t + 4) * hop]), **oracle_kwargs(mine))
    assert fwd.shape == (2, 1, t * hop) and inf.shape == (2, 1, (t + 4) * hop)
    rec.check("forward", fwd, lambda: reference()["forward"])
    rec.check("inference", inf, lambda: reference()["inference"])


@pytest.mark.parametrize("weight_norm", [True, False])
def test_pwgan_state_dict_layout_matches_reference(R, rec, weight_norm):
    want = rec.value("layout", lambda: layout(R(use_weight_norm=weight_norm).state_dict()))
    got = layout(ParallelWaveganGenerator(use_weight_norm=weight_norm).state_dict())
    assert [(k, s, d) for k, s, d, _ in got] == [(k, s, d) for k, s, d, _ in want]
    if weight_norm:
        assert len(got) == 349
        assert "upsample_net.upsample.up_layers.7.parametrizations.weight.original1" in [k for k, *_ in got]


def test_pwgan_config_and_setup_generator_surface(R, rec):
    mine = {f.name: getattr(V.ParallelWaveganConfig(), f.name) for f in dataclasses.fields(V.ParallelWaveganConfig)
            if f.name != "audio"}

    def ref_fields():
        cls = importlib.import_module("TTS.vocoder.configs.parallel_wavegan_config").ParallelWaveganConfig
        return {k: getattr(cls(), k) for k in mine}

    assert mine == rec.value("fields", ref_fields)

    def ref_shapes():
        cfg = importlib.import_module("TTS.vocoder.configs.parallel_wavegan_config").ParallelWaveganConfig()
        gen = importlib.import_module("TTS.vocoder.models").setup_generator(cfg)
        gan = importlib.import_module("TTS.vocoder.models.gan").GAN(cfg)
        return ([(k, tuple(v.shape)) for k, v in gen.state_dict().items()],
                [(k, tuple(v.shape)) for k, v in gan.state_dict().items() if k.startswith("model_g.")])

    gen_want, gan_want = rec.value("shapes", ref_shapes)
    g = V.setup_generator(V.ParallelWaveganConfig())
    assert type(g).__name__ == "ParallelWaveganGenerator"
    assert [(k, tuple(v.shape)) for k, v in g.state_dict().items()] == gen_want
    gan = V.setup_model(V.ParallelWaveganConfig())
    assert type(gan).__name__ == "GAN"
    assert [(k, tuple(v.shape)) for k, v in gan.state_dict().items()] == gan_want
    # MelGAN params have no `stacks`: the reference's KeyError, which is also a NotImplementedError here
    with pytest.raises(KeyError):
        V.setup_generator(V.MelganConfig(generator_model="parallel_wavegan_generator"))


def test_legacy_weight_norm_checkpoint(tmp_path):
    model = ParallelWaveganGenerator(num_res_blocks=4, stacks=2, upsample_factors=[2, 3])
    sd = seeded_state_dict(layout(model.state_dict()), 9)
    legacy = {k.replace(".parametrizations.weight.original0", ".weight_g")
               .replace(".parametrizations.weight.original1", ".weight_v"): v for k, v in sd.items()}
    assert any(k.endswith(".weight_g") for k in legacy)
    path = tmp_path / "pwgan.pth"
    torch.save({"model": legacy}, path)
    fresh = ParallelWaveganGenerator(num_res_blocks=4, stacks=2, upsample_factors=[2, 3])
    fresh.load_checkpoint(None, str(path), eval=False)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, sd[k]), k
    c = torch.randn(1, 80, 5)
    noise = torch.randn(1, 1, 30)
    kw = oracle_kwargs(fresh)
    assert torch.equal(PO.generator(legacy, c, noise, **kw), PO.generator(sd, c, noise, **kw))
    fresh.load_checkpoint(None, str(path), eval=True)
    assert not fresh.training
    assert all(not k.endswith(("original0", "original1")) for k in fresh.state_dict())
    assert torch.equal(fresh.conv_layers[1].conv.weight, PO.conv_weight(sd, "conv_layers.1.conv"))


def test_num_mels_other_than_80_error_type(R, rec):
    """ConvUpsample keeps 80 channels whatever aux_channels is: the reference fails in its convs (RuntimeError)."""
    c = torch.randn(1, 64, 5)

    def ref_error():
        try:
            R(aux_channels=64, num_res_blocks=2, stacks=1)(c)
        except Exception as e:  # noqa: BLE001 - the exception type is the result
            return type(e).__name__
        return None

    assert rec.value("error", ref_error) == "RuntimeError"
    m = ParallelWaveganGenerator(aux_channels=64, num_res_blocks=2, stacks=1)
    assert tuple(m.conv_layers[0].conv1x1_aux.weight.shape) == (128, 64, 1)
    assert tuple(m.upsample_net.conv_in.weight.shape) == (80, 80, 1)
    # the drop-in's own check, before any device is needed (on a CUDA tensor too, where one is present)
    inputs = [c] + ([c.cuda()] if torch.cuda.is_available() else [])
    for x in inputs:
        with pytest.raises(RuntimeError, match="takes 80 channels"):
            m(x)
    cfg = V.ParallelWaveganConfig()
    cfg.audio.num_mels = 64
    for x in inputs:
        with pytest.raises(RuntimeError, match="takes 80 channels"):
            V.setup_generator(cfg)(x)


@pytest.mark.parametrize("field,value", [("res_channels", 32), ("skip_channels", 128), ("gate_channels", 64),
                                         ("kernel_size", 5)])
def test_shapes_the_kernel_does_not_take(field, value):
    with pytest.raises(NotImplementedError, match=field):
        ParallelWaveganGenerator(**{field: value})


def test_no_cpu_path():
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    m = ParallelWaveganGenerator(num_res_blocks=2, stacks=1)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(torch.randn(1, 80, 5))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.inference(torch.randn(1, 80, 5))
