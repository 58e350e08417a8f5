"""Streaming decode (``HifiganGenerator.forward_window`` / ``Vits.inference_stream``): the waveform of any window of
decoder-input frames must be BIT-IDENTICAL to the same samples of the one-shot call -- checked with torch.equal against
the one-shot CUDA path (which the other tests tie to the oracle) -- and a window call must touch no other sample."""
import math

import pytest
import torch

from tts_b200 import _lib

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _decoder(cond=0):
    from tts_b200.hifigan import HifiganGenerator
    return HifiganGenerator(in_channels=192, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
                            resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4],
                            upsample_initial_channel=512, upsample_factors=[8, 8, 2, 2], inference_padding=0,
                            cond_channels=cond, conv_pre_weight_norm=False, conv_post_weight_norm=False,
                            conv_post_bias=False).eval()


def _poison_workspace(m, z):
    """Fill the decoder's cached workspace with NaN: a window must not read what earlier calls left there."""
    b, _, t = z.shape
    h = m._ensure_handle(z.device)
    nbytes = _lib.lib().b200tts_hifigan_workspace_bytes(h, b, t)
    _lib.workspace(z.device, nbytes, "hifigan").fill_(255)          # 0xFFFFFFFF is a NaN


def _stream(m, z, chunk, g=None, lengths=None, peak=None):
    """Consecutive windows of `chunk` frames into one NaN-prefilled buffer."""
    b, _, t = z.shape
    hop = m.hop
    out = torch.full((b, m._cfg["out_channels"], t * hop), NAN, device=z.device)
    for f0 in range(0, t, chunk):
        f1 = min(t, f0 + chunk)
        _poison_workspace(m, z)
        v = m.forward_window(z, g, start=f0, end=f1, lengths=lengths, out=out, peak=peak)
        assert v.shape[-1] == (f1 - f0) * hop and v.data_ptr() == out[..., f0 * hop:].data_ptr()
    return out


def _masked_z(b, t, lens, c=192):
    if lens is None:
        return torch.randn(b, c, t).cuda()
    mask = (torch.arange(t)[None, :] < torch.tensor(lens)[:, None]).float().unsqueeze(1)
    return (torch.randn(b, c, t) * mask).cuda()                       # what Vits feeds: z * y_mask


@pytest.mark.parametrize("b,t,lens,chunk,cond", [
    (6, 150, [150, 97, 64, 33, 2, 1], 32, 0),
    (3, 64, None, 7, 0),
    (2, 301, [17, 301], 1, 0),          # T % 4 != 0: the stage-0 tensors are re-pitched
    (1, 90, None, 16, 0),               # T < 128: conv_pre / ups[0] run on the FP32-FMA kernel
    (3, 90, [90, 41, 12], 16, 256),     # speaker conditioning
])
def test_decoder_windows_equal_full_call(b, t, lens, chunk, cond):
    torch.manual_seed(b * 1000 + t + chunk)
    m = _decoder(cond).cuda()
    z = _masked_z(b, t, lens)
    g = torch.randn(b, cond, 1).cuda() if cond else None
    full = m(z, g)
    got = _stream(m, z, chunk, g)
    assert torch.equal(got, full)
    if lens is not None:
        lt = torch.tensor(lens).cuda()
        full_r = m(z, g, lengths=lt)
        got_r = _stream(m, z, chunk, g, lengths=lt)
        assert torch.equal(got_r, full_r)                            # zeros past each row's end included


def test_single_window_touches_only_its_samples():
    torch.manual_seed(11)
    m = _decoder().cuda()
    z = _masked_z(2, 150, None)
    full = m(z)
    f0, f1 = 40, 77
    for lengths in (None, torch.tensor([150, 61]).cuda()):
        want = full if lengths is None else m(z, lengths=lengths)
        out = torch.full_like(full, NAN)
        _poison_workspace(m, z)
        v = m.forward_window(z, start=f0, end=f1, lengths=lengths, out=out)
        assert torch.equal(v, want[..., f0 * 256: f1 * 256])
        assert torch.isnan(out[..., : f0 * 256]).all() and torch.isnan(out[..., f1 * 256:]).all()


@pytest.mark.parametrize("ragged", [False, True])
def test_window_dispatch_matches_full_call(ragged):
    torch.manual_seed(12)
    m = _decoder().cuda()
    z = _masked_z(4, 200, [200, 150, 80, 9])
    lengths = torch.tensor([200, 150, 80, 9]).cuda() if ragged else None
    with _lib.dispatch_log() as full:
        m(z, lengths=lengths)
    assert full.names
    out = torch.empty(4, 1, 200 * 256, device="cuda")
    for f0 in range(0, 200, 48):
        with _lib.dispatch_log() as win:
            m.forward_window(z, start=f0, end=min(200, f0 + 48), lengths=lengths, out=out)
        assert win.names == full.names, f0


def test_other_geometry_streams_exactly():
    """hop 6 (not a multiple of 4) and two output channels: conv_post on the FMA tanh epilogue, peak by its own pass."""
    from tts_b200.hifigan import HifiganGenerator
    from tts_b200.vocoder import new_peak
    torch.manual_seed(13)
    m = HifiganGenerator(in_channels=20, out_channels=2, resblock_type="1", resblock_dilation_sizes=[[1, 2], [2, 6]],
                         resblock_kernel_sizes=[3, 5], upsample_kernel_sizes=[7, 4], upsample_initial_channel=64,
                         upsample_factors=[3, 2]).eval().cuda()
    assert m.hop == 6
    z = torch.randn(3, 20, 101).cuda()
    p_full, p_win = new_peak(z.device), new_peak(z.device)
    full = m(z, peak=p_full)
    assert full.shape[-1] == 101 * 6
    for chunk in (1, 10, 33):
        got = _stream(m, z, chunk, peak=p_win)
        assert torch.equal(got, full), chunk
    assert torch.equal(p_win, p_full)


def test_bad_window_or_geometry_raises():
    from tts_b200.hifigan import HifiganGenerator
    m = HifiganGenerator(in_channels=20, out_channels=2, resblock_type="1", resblock_dilation_sizes=[[1, 2], [2, 6]],
                         resblock_kernel_sizes=[3, 5], upsample_kernel_sizes=[7, 3], upsample_initial_channel=64,
                         upsample_factors=[3, 2]).eval().cuda()
    z = torch.randn(2, 20, 29).cuda()
    with pytest.raises(ValueError, match="multiply the length"):
        m.forward_window(z, start=0, end=10)
    d = _decoder().cuda()
    z = torch.randn(1, 192, 20).cuda()
    for s, e in ((5, 5), (-1, 4), (0, 21), (12, 3)):
        with pytest.raises(ValueError, match="window"):
            d.forward_window(z, start=s, end=e)


def test_peak_over_windows_equals_full_call():
    from tts_b200.vocoder import new_peak
    torch.manual_seed(14)
    m = _decoder().cuda()
    z = _masked_z(3, 130, [130, 70, 20])
    for lengths in (None, torch.tensor([130, 70, 20]).cuda()):
        p_full, p_win = new_peak(z.device), new_peak(z.device)
        full = m(z, peak=p_full, lengths=lengths)
        got = _stream(m, z, 32, lengths=lengths, peak=p_win)
        assert torch.equal(got, full)
        assert torch.equal(p_win, p_full)


def _vits(num_speakers=9):
    from tts_b200.vits import Vits, VitsArgs, VitsConfig
    torch.manual_seed(8)
    cfg = VitsConfig(model_args=VitsArgs(use_speaker_embedding=True, num_speakers=num_speakers))
    m = Vits(cfg).eval()
    gen = torch.Generator().manual_seed(1)
    for _, p in m.named_parameters():
        if float(p.detach().abs().sum()) == 0.0:
            p.data.copy_(torch.randn(p.shape, generator=gen) * 0.05)
    return m.cuda()


def _check_stream(m, tok, aux, noise, chunk_frames):
    store = {}

    def prior(shape):
        if "n" not in store:
            store["n"] = torch.randn(shape, generator=torch.Generator().manual_seed(2)).cuda()
        return store["n"]

    full = m.inference(tok, aux, sdp_noise=noise, prior_noise=prior)
    chunks = list(m.inference_stream(tok, aux, chunk_frames=chunk_frames, sdp_noise=noise, prior_noise=prior))
    t_dec = full["y_mask"].shape[-1]
    assert len(chunks) == math.ceil(t_dec / chunk_frames)
    start = 0
    for c in chunks:
        assert c["start"] == start
        assert torch.equal(c["wav_lengths"], full["wav_lengths"])
        start += c["model_outputs"].shape[-1]
    wav = torch.cat([c["model_outputs"] for c in chunks], dim=-1)
    assert torch.equal(wav, full["model_outputs"])
    return full


@pytest.mark.parametrize("trim", [False, True])
def test_vits_inference_stream_equals_inference(trim):
    m = _vits()
    m.trim_padding = trim
    lens = torch.tensor([64, 50, 33, 20, 11, 64, 5, 41])
    gen = torch.Generator().manual_seed(3)
    tok = (torch.randint(0, 100, (8, 64), generator=gen) * (torch.arange(64)[None, :] < lens[:, None])).cuda()
    aux = {"x_lengths": lens.cuda(), "speaker_ids": torch.randint(0, 9, (8,), generator=gen).cuda()}
    noise = torch.randn(8, 2, 64, generator=gen)
    full = _check_stream(m, tok, aux, noise, 24)
    wl = full["wav_lengths"].tolist()
    assert min(wl) < max(wl)                                        # the batch really is ragged


@pytest.mark.parametrize("length_scale", [1.0, 3.0])
def test_stream_at_benchmark_scale(length_scale):
    """cfg2: 32 utterances x 64 tokens, the default VitsConfig decoder, ragged windows as bench.py runs it."""
    from tts_b200.vits import Vits, VitsConfig
    torch.manual_seed(1234)
    m = Vits(VitsConfig()).eval().cuda()
    m.trim_padding = True
    m.length_scale = length_scale
    gen = torch.Generator().manual_seed(4321)
    tok = torch.randint(0, 100, (32, 64), generator=gen).cuda()
    aux = {"x_lengths": torch.full((32,), 64, dtype=torch.int64).cuda()}
    noise = torch.randn(32, 2, 64, generator=gen).cuda()
    _check_stream(m, tok, aux, noise, 32)
