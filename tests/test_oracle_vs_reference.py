"""Runs the oracle port side by side with the UNMODIFIED reference modules at FULL model sizes.  Where the reference
tree is absent the reference's results recorded under tests/golden/reference/ stand in for it (oracle/ref_golden.py)."""
import pytest
import torch

import ref_import
import vits_oracle as O
from ref_golden import Recorded, layout, seeded_state_dict


@pytest.fixture(scope="module")
def R():
    return ref_import.load() if ref_import.available() else None


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def _once(fn):
    cache = []

    def get():
        if not cache:
            cache.append(fn())
        return cache[0]
    return get


def _loaded(module, sd):
    module.load_state_dict(sd)
    return module.eval()


@torch.no_grad()
def test_hifigan_full_width(R, rec):
    mk = _once(lambda: R["hifigan"].HifiganGenerator(192, 1, "1", [[1, 3, 5]] * 3, [3, 7, 11], [16, 16, 4, 4], 512,
                                                     [8, 8, 2, 2], inference_padding=0, cond_channels=256,
                                                     conv_pre_weight_norm=False, conv_post_weight_norm=False,
                                                     conv_post_bias=False).eval())
    sd = seeded_state_dict(rec.value("layout", lambda: layout(mk().state_dict())), 0)
    gen = torch.Generator().manual_seed(0)
    x, g = torch.randn(1, 192, 6, generator=gen), torch.randn(1, 256, 1, generator=gen)
    rec.check("y", O.hifigan_forward(sd, x, g), lambda: _loaded(mk(), sd)(x, g))


@torch.no_grad()
def test_vits_stack_full_width(R, rec):
    gen = torch.Generator().manual_seed(1)
    te = _once(lambda: R["networks"].TextEncoder(100, 192, 192, 768, 2, 6, 3, 0.1))
    te_sd = seeded_state_dict(rec.value("te_layout", lambda: layout(te().state_dict())), 1)
    tok, lens = torch.randint(0, 100, (3, 21), generator=gen), torch.tensor([21, 13, 5])
    got = O.text_encoder(te_sd, tok, lens)
    want = _once(lambda: _loaded(te(), te_sd)(tok, lens))
    for i, t in enumerate(got):
        rec.check(f"te{i}", t, lambda i=i: want()[i])
    g = torch.randn(3, 256, 1, generator=gen)
    sdp = _once(lambda: R["sdp"].StochasticDurationPredictor(192, 192, 3, 0.5, 4, cond_channels=256))
    sdp_sd = seeded_state_dict(rec.value("sdp_layout", lambda: layout(sdp().state_dict())), 2)
    torch.manual_seed(9)
    noise = torch.randn(3, 2, 21)

    def sdp_ref():
        m = _loaded(sdp(), sdp_sd)
        torch.manual_seed(9)              # the reference draws the same noise inside forward
        return m(got[0], got[3], g=g, reverse=True, noise_scale=1.0)
    rec.check("sdp", O.sdp_reverse(sdp_sd, got[0], got[3], noise, g=g), sdp_ref)
    fl = _once(lambda: R["networks"].ResidualCouplingBlocks(192, 192, 5, 1, 4, cond_channels=256))
    fl_sd = seeded_state_dict(rec.value("flow_layout", lambda: layout(fl().state_dict())), 3)
    z = torch.randn(3, 192, 40, generator=gen)
    mask = O.sequence_mask(torch.tensor([40, 22, 3]), 40).unsqueeze(1).float()
    rec.check("flow", O.flow_forward(fl_sd, z, mask, g, reverse=True),
              lambda: _loaded(fl(), fl_sd)(z, mask, g=g, reverse=True))


def test_mas_cfg4_shape_against_compiled_reference(R, rec):
    import numpy as np

    assert rec.value("cython", lambda: R["helpers"].CYTHON)
    rng = np.random.RandomState(0)
    v = torch.from_numpy(rng.randn(8, 200, 1000).astype(np.float32))
    t_x = torch.from_numpy(rng.randint(100, 201, size=8))
    t_y = torch.tensor([int(rng.randint(5 * int(a) if 5 * int(a) <= 1000 else 1000, 1001)) for a in t_x])
    mask = ((torch.arange(200)[None, :, None] < t_x[:, None, None]) &
            (torch.arange(1000)[None, None, :] < t_y[:, None, None])).float()
    got = O.maximum_path(v, mask, impl="c")
    rec.check("path", got, lambda: R["helpers"].maximum_path(v, mask))
    if ref_import.load_ref_mas_core() is not None:       # the compiled reference kernel, where build() made it
        assert torch.equal(O.maximum_path(v, mask, impl="ref"), got)


@torch.no_grad()
def test_voice_conversion_stack_full_width(R, rec):
    """Posterior encoder, flow forward and the deterministic duration predictor at VITS width vs the reference."""
    gen = torch.Generator().manual_seed(4)
    pe = _once(lambda: R["networks"].PosteriorEncoder(513, 192, 192, 5, 1, 16, cond_channels=256))
    pe_sd = seeded_state_dict(rec.value("pe_layout", lambda: layout(pe().state_dict())), 4)
    y, g = torch.randn(2, 513, 33, generator=gen).abs(), torch.randn(2, 256, 1, generator=gen)
    lens = torch.tensor([33, 12])
    torch.manual_seed(5)
    noise = torch.randn(2, 192, 33)
    got = O.posterior_encoder(pe_sd, y, lens, g=g, noise=noise)

    def pe_ref():
        m = _loaded(pe(), pe_sd)
        torch.manual_seed(5)              # the reference draws randn_like(mean) inside forward
        return m(y, lens, g=g)
    want = _once(pe_ref)
    for i, t in enumerate(got):
        rec.check(f"pe{i}", t, lambda i=i: want()[i])
    fl = _once(lambda: R["networks"].ResidualCouplingBlocks(192, 192, 5, 1, 4, cond_channels=256))
    fl_sd = seeded_state_dict(rec.value("flow_layout", lambda: layout(fl().state_dict())), 5)
    rec.check("flow", O.flow_forward(fl_sd, got[0], got[3], g, reverse=False),
              lambda: _loaded(fl(), fl_sd)(got[0], got[3], g=g))
    dp = _once(lambda: R["duration_predictor"].DurationPredictor(192, 256, 3, 0.5, cond_channels=256))
    dp_sd = seeded_state_dict(rec.value("dp_layout", lambda: layout(dp().state_dict())), 6)
    x = torch.randn(2, 192, 17, generator=gen)
    xm = O.sequence_mask(torch.tensor([17, 6]), 17).unsqueeze(1).float()
    rec.check("dp", O.duration_predictor(dp_sd, x, xm, g=g), lambda: _loaded(dp(), dp_sd)(x, xm, g=g), atol=1e-6)


def test_drop_in_state_dict_keys_match_reference(R, rec):
    """The Python mirror must load reference checkpoints unchanged: same state_dict keys and shapes."""
    from tts_b200 import layers as L
    from tts_b200.hifigan import HifiganGenerator

    def keys(m):
        return {k: tuple(v.shape) for k, v in m.state_dict().items()}

    kw = dict(in_channels=192, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
              resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512,
              upsample_factors=[8, 8, 2, 2], inference_padding=0, cond_channels=256, conv_pre_weight_norm=False,
              conv_post_weight_norm=False, conv_post_bias=False)
    pairs = [
        ("TextEncoder", lambda: R["networks"].TextEncoder(50, 192, 192, 768, 2, 6, 3, 0.1, language_emb_dim=4),
         L.TextEncoder(50, 192, 192, 768, 2, 6, 3, 0.1, language_emb_dim=4)),
        ("ResidualCouplingBlocks", lambda: R["networks"].ResidualCouplingBlocks(192, 192, 5, 1, 4, cond_channels=256),
         L.ResidualCouplingBlocks(192, 192, 5, 1, 4, cond_channels=256)),
        ("PosteriorEncoder", lambda: R["networks"].PosteriorEncoder(513, 192, 192, 5, 1, 16, cond_channels=256),
         L.PosteriorEncoder(513, 192, 192, 5, 1, 16, cond_channels=256)),
        ("StochasticDurationPredictor",
         lambda: R["sdp"].StochasticDurationPredictor(192, 192, 3, 0.5, 4, cond_channels=256, language_emb_dim=4),
         L.StochasticDurationPredictor(192, 192, 3, 0.5, 4, cond_channels=256, language_emb_dim=4)),
        ("DurationPredictor",
         lambda: R["duration_predictor"].DurationPredictor(192, 256, 3, 0.5, cond_channels=256, language_emb_dim=4),
         L.DurationPredictor(192, 256, 3, 0.5, cond_channels=256, language_emb_dim=4)),
        ("HifiganGenerator", lambda: R["hifigan"].HifiganGenerator(**kw), HifiganGenerator(**kw)),
    ]
    for name, ref, ours in pairs:
        assert rec.value(name, lambda: keys(ref())) == keys(ours), name
