"""UnivNet without a GPU: the CPU restatement (tests/univnet_oracle.py) is pinned ``torch.equal`` to the unmodified
reference generator on the reference's own seeded noise draws -- live where the reference tree imports, through the
results recorded under tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest
tests/test_univnet_oracle_cpu.py`` where the reference is present) -- and the drop-in's surface (config defaults,
state-dict layout, setup_generator / GAN / setup_model, legacy weight-norm checkpoints, error behaviour) is checked
against it."""
import dataclasses
import importlib

import pytest
import torch

import ref_import
import univnet_oracle as UO
from ref_golden import Recorded, layout, seeded_state_dict
from tts_b200 import vocoder as V
from tts_b200.univnet import UnivnetGenerator

REF_MODULE = "TTS.vocoder.models.univnet_generator"

DEFAULT = dict(in_channels=64, out_channels=1, hidden_channels=32, cond_channels=80, upsample_factors=[8, 8, 4],
               lvc_layers_each_block=4, lvc_kernel_size=3, kpnet_hidden_channels=64, kpnet_conv_size=3, dropout=0.0)

# name -> (constructor overrides, frames T)
CASES = {
    "default_T1": (dict(), 1),
    "default_T3": (dict(), 3),
    "default_T40": (dict(), 40),
    "factors_3_5_4": (dict(upsample_factors=[3, 5, 4]), 4),
    "layers_2": (dict(lvc_layers_each_block=2), 3),
    "kpnet_conv_size_5": (dict(kpnet_conv_size=5), 3),
    "cond_channels_100": (dict(cond_channels=100), 3),
    "hidden_16": (dict(hidden_channels=16), 3),
    "no_weight_norm": (dict(use_weight_norm=False), 3),
}


def params(over):
    p = dict(DEFAULT)
    p.update(over)
    return p


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    return importlib.import_module(REF_MODULE).UnivnetGenerator


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def oracle_kwargs(p):
    return dict(upsample_factors=tuple(p["upsample_factors"]), layers=p["lvc_layers_each_block"])


@pytest.mark.parametrize("case", list(CASES))
def test_univnet_oracle_equals_reference(R, rec, case):
    over, t = CASES[case]
    p = params(over)
    mine = UnivnetGenerator(**p)
    sd = seeded_state_dict(layout(mine.state_dict()), 5)
    c = torch.randn(2, p["cond_channels"], t, generator=torch.Generator().manual_seed(1))
    hop = mine.upsample_scale
    ref = {}

    def reference():
        if not ref:
            net = R(**p).eval()
            net.load_state_dict(sd)
            with torch.no_grad():
                torch.manual_seed(21)
                ref["forward"] = net(c.clone())
                torch.manual_seed(22)
                ref["inference"] = net.inference(c.clone())
        return ref

    torch.manual_seed(21)                  # the reference's draw: torch.randn([B, in_channels, T]) on the CPU generator
    fwd = UO.generator(sd, c, torch.randn([2, p["in_channels"], t]), **oracle_kwargs(p))
    torch.manual_seed(22)
    torch.randn([2, p["in_channels"], t])  # inference's own draw, discarded; forward then draws again
    inf = UO.generator(sd, c, torch.randn([2, p["in_channels"], t]), **oracle_kwargs(p))
    assert fwd.shape == (2, 1, t * hop) and inf.shape == (2, 1, t * hop)
    rec.check("forward", fwd, lambda: reference()["forward"])
    rec.check("inference", inf, lambda: reference()["inference"])


@pytest.mark.parametrize("weight_norm", [True, False])
def test_univnet_state_dict_layout_matches_reference(R, rec, weight_norm):
    want = rec.value("layout", lambda: layout(R(**DEFAULT, use_weight_norm=weight_norm).state_dict()))
    got = layout(UnivnetGenerator(**DEFAULT, use_weight_norm=weight_norm).state_dict())
    assert [(k, s, d) for k, s, d, _ in got] == [(k, s, d) for k, s, d, _ in want]
    keys = [k for k, *_ in got]
    assert ("lvc_blocks.2.kernel_predictor.kernel_conv.parametrizations.weight.original1" in keys) == weight_norm
    assert "lvc_blocks.0.upsample.weight" in keys   # ConvTranspose1d takes no weight norm


def ref_config():
    """The reference's UnivnetConfig.__post_init__ calls a super().__post_init__ that none of its bases defines, so the
    class cannot be instantiated as it stands; this subclass runs the rest of its __post_init__ (cond_channels =
    audio.num_mels) without that call."""
    cls = importlib.import_module("TTS.vocoder.configs.univnet_config").UnivnetConfig

    @dataclasses.dataclass
    class UnivnetConfig(cls):  # same name: the reference dispatches on the class name
        def __post_init__(self):
            self.generator_model_params["cond_channels"] = self.audio.num_mels

    return UnivnetConfig()


def test_univnet_config_and_setup_generator_surface(R, rec):
    mine = {f.name: getattr(V.UnivnetConfig(), f.name) for f in dataclasses.fields(V.UnivnetConfig) if f.name != "audio"}

    def ref_fields():
        cfg = ref_config()
        return {k: getattr(cfg, k) for k in mine}

    assert mine == rec.value("fields", ref_fields)
    cfg = V.UnivnetConfig()
    cfg.audio.num_mels = 100
    cfg.__post_init__()
    assert cfg.generator_model_params["cond_channels"] == 100

    def ref_shapes():
        cfg = ref_config()
        gen = importlib.import_module("TTS.vocoder.models").setup_generator(cfg)
        gan = importlib.import_module("TTS.vocoder.models.gan").GAN(cfg)
        return ([(k, tuple(v.shape)) for k, v in gen.state_dict().items()],
                [(k, tuple(v.shape)) for k, v in gan.state_dict().items() if k.startswith("model_g.")])

    gen_want, gan_want = rec.value("shapes", ref_shapes)
    g = V.setup_generator(V.UnivnetConfig())
    assert type(g).__name__ == "UnivnetGenerator"
    assert [(k, tuple(v.shape)) for k, v in g.state_dict().items()] == gen_want
    gan = V.setup_model(V.UnivnetConfig())
    assert type(gan).__name__ == "GAN"
    assert [(k, tuple(v.shape)) for k, v in gan.state_dict().items()] == gan_want


def test_univnet_bad_params_error_type(R, rec):
    """MelGAN params given to univnet_generator: the reference's TypeError from UnivnetGenerator(**params)."""
    def ref_error():
        cfg = importlib.import_module("TTS.vocoder.configs.melgan_config").MelganConfig(generator_model="univnet_generator")
        try:
            importlib.import_module("TTS.vocoder.models").setup_generator(cfg)
        except Exception as e:  # noqa: BLE001 - the exception type is the result
            return type(e).__name__
        return None

    assert rec.value("error", ref_error) == "TypeError"
    with pytest.raises(TypeError):
        V.setup_generator(V.MelganConfig(generator_model="univnet_generator"))
    with pytest.raises(V.GeneratorParamsTypeError):
        V.setup_generator(V.MelganConfig(generator_model="univnet_generator"))


def test_gan_load_checkpoint(tmp_path):
    cfg = V.UnivnetConfig()
    gan = V.GAN(cfg)
    sd = seeded_state_dict(layout(gan.state_dict()), 3)
    path = tmp_path / "univnet_gan.pth"
    torch.save({"model": sd}, path)
    fresh = V.GAN(V.UnivnetConfig())
    fresh.load_checkpoint(cfg, str(path), eval=True)
    assert not fresh.training
    assert all(not k.endswith(("original0", "original1")) for k in fresh.state_dict())
    w = fresh.model_g.lvc_blocks[1].kernel_predictor.kernel_conv.weight
    assert torch.equal(w, UO.conv_weight({k[len("model_g."):]: v for k, v in sd.items()},
                                         "lvc_blocks.1.kernel_predictor.kernel_conv"))


def test_legacy_weight_norm_checkpoint(tmp_path):
    p = params(dict(upsample_factors=[2, 3], lvc_layers_each_block=2, kpnet_hidden_channels=16))
    model = UnivnetGenerator(**p)
    sd = seeded_state_dict(layout(model.state_dict()), 9)
    legacy = {k.replace(".parametrizations.weight.original0", ".weight_g")
               .replace(".parametrizations.weight.original1", ".weight_v"): v for k, v in sd.items()}
    assert any(k.endswith(".weight_g") for k in legacy)
    path = tmp_path / "univnet.pth"
    torch.save({"model": legacy}, path)
    fresh = UnivnetGenerator(**p)
    fresh.load_checkpoint(None, str(path), eval=False)
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, sd[k]), k
    c, noise = torch.randn(1, 80, 3), torch.randn(1, 64, 3)
    kw = oracle_kwargs(p)
    assert torch.equal(UO.generator(legacy, c, noise, **kw), UO.generator(sd, c, noise, **kw))
    fresh.load_checkpoint(None, str(path), eval=True)
    assert not fresh.training
    assert all(not k.endswith(("original0", "original1")) for k in fresh.state_dict())


@pytest.mark.parametrize("field,value", [("hidden_channels", 16), ("lvc_kernel_size", 5),
                                         ("kpnet_hidden_channels", 40)])
def test_shapes_the_kernels_do_not_take(field, value):
    """The module builds (its state dict is the reference's); running it on the GPU path raises, naming the field."""
    m = UnivnetGenerator(**params({field: value})).eval()
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    with pytest.raises(NotImplementedError, match=field):
        m.to(dev)(torch.randn(1, 80, 2, device=dev))


def test_dropout_in_training_mode():
    m = UnivnetGenerator(**params(dict(dropout=0.1)))
    assert m.training
    with pytest.raises(NotImplementedError, match="dropout"):
        m(torch.randn(1, 80, 2))


def test_no_cpu_path():
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    m = UnivnetGenerator(**DEFAULT).eval()
    c = torch.randn(1, 80, 2)
    state = torch.get_rng_state()
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(c)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.inference(c)
    assert torch.equal(state, torch.get_rng_state())   # a failing call draws nothing
