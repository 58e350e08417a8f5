"""Every engine's workspace size is exactly what its call uses.

``_lib.workspace`` is replaced by a fake that hands each module the first ``nbytes`` bytes of a fresh buffer followed by
64 KiB of 0xA5 bytes.  With the size the module asked for, the call must give what it gives through the real
``_lib.workspace`` (bit for bit) and leave the 0xA5 tail alone; one byte less must raise ``RuntimeError`` before the
library launches anything.  Shapes: B = 1 and 3, frame counts that are not a multiple of 4, ragged lengths where the
entry point takes them.  PWGAN's ``layer`` and UnivNet's ``predict`` have no module call and go through the C ABI.
"""
import ctypes

import numpy as np
import pytest
import torch

from tts_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TAIL = 64 * 1024


def lens_for(b, t):
    return torch.tensor([t, t - 6, 3][:b], device=DEV)


def mask_for(lens, t):
    return (torch.arange(t, device=DEV)[None, :] < lens[:, None]).float().unsqueeze(1)


def hifigan(window=False):
    from tts_b200.hifigan import HifiganGenerator
    m = HifiganGenerator(in_channels=20, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
                         resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4],
                         upsample_initial_channel=64, upsample_factors=[8, 8, 2, 2], cond_channels=8).eval().to(DEV)

    def call(b, t=37):
        x, g, lens = torch.randn(b, 20, t, device=DEV), torch.randn(b, 8, 1, device=DEV), lens_for(b, t)
        if window:
            return m.forward_window(x, g, start=5, end=21, lengths=lens)
        return m(x, g, lengths=lens)
    return call


def flow(reverse):
    from tts_b200.layers import ResidualCouplingBlocks
    m = ResidualCouplingBlocks(8, 16, 5, 1, 2, num_flows=2, cond_channels=4).eval().to(DEV)

    def call(b, t=37):
        lens = lens_for(b, t)
        mask = mask_for(lens, t)
        return m(torch.randn(b, 8, t, device=DEV) * mask, mask, torch.randn(b, 4, 1, device=DEV), reverse=reverse,
                 lengths=lens)
    return call


def text_encoder():
    from tts_b200.layers import TextEncoder
    m = TextEncoder(30, 8, 16, 32, 2, 2, 3, 0.1).eval().to(DEV)
    return lambda b, t=23: m(torch.randint(1, 30, (b, t), device=DEV), lens_for(b, t))


def sdp():
    from tts_b200.layers import StochasticDurationPredictor
    m = StochasticDurationPredictor(16, 16, 3, 0.5, 4, cond_channels=4).eval().to(DEV)

    def call(b, t=23):
        mask = mask_for(lens_for(b, t), t)
        return m(torch.randn(b, 16, t, device=DEV), mask, g=torch.randn(b, 4, 1, device=DEV), reverse=True)
    return call


def posterior():
    from tts_b200.layers import PosteriorEncoder
    m = PosteriorEncoder(20, 8, 16, 5, 1, 4, cond_channels=4).eval().to(DEV)
    return lambda b, t=37: m(torch.randn(b, 20, t, device=DEV), lens_for(b, t), torch.randn(b, 4, 1, device=DEV))


def duration_predictor():
    from tts_b200.layers import DurationPredictor
    m = DurationPredictor(16, 32, 3, 0.5, cond_channels=4).eval().to(DEV)
    return lambda b, t=23: m(torch.randn(b, 16, t, device=DEV), mask_for(lens_for(b, t), t),
                             torch.randn(b, 4, 1, device=DEV))


def speaker_encoder(stage=None):
    from tts_b200.encoder import ResNetSpeakerEncoder
    audio = dict(fft_size=512, win_length=400, hop_length=160, sample_rate=16000, preemphasis=0.97, num_mels=64)
    m = ResNetSpeakerEncoder(encoder_type="ASP", log_input=True, use_torch_spec=True, audio_config=audio).eval().to(DEV)

    def call(b, t=4803):
        x = torch.randn(b, t, device=DEV) * 0.1
        return m(x) if stage is None else m.forward_features(x, stage)
    return call


def tts(kind):
    if kind == "glow_tts":
        from tts_b200.glow_tts import GlowTTS, GlowTTSConfig
        m, aux = GlowTTS(GlowTTSConfig(num_chars=30)), {}
    elif kind == "forward_tts":
        from tts_b200.forward_tts import FastPitchConfig, ForwardTTS, ForwardTTSArgs
        m, aux = ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=30))), {}
    elif kind == "overflow":
        from tts_b200 import overflow as OV
        m, aux = OV.Overflow(OV.OverflowConfig(num_chars=30)), {"sampling_temp": 0.0, "max_sampling_time": 30}
    elif kind == "tacotron2":
        from tts_b200 import tacotron2 as T2
        m, aux = T2.Tacotron2(T2.Tacotron2Config(num_chars=30, max_decoder_steps=30)), {}
    else:
        from tts_b200 import tacotron as T1
        m, aux = T1.Tacotron(T1.TacotronConfig(num_chars=30, max_decoder_steps=30)), {}
    m.eval().to(DEV)
    return lambda b, t=23: m.inference(torch.randint(1, 30, (b, t), device=DEV), dict(aux, x_lengths=lens_for(b, t)))


def vocoder(kind):
    from tts_b200 import melgan, pwgan, univnet
    m = {"melgan": lambda: melgan.MelganGenerator(base_channels=64, num_res_blocks=2),
         "multiband_melgan": lambda: melgan.MultibandMelganGenerator(base_channels=64, num_res_blocks=2),
         "pwgan": lambda: pwgan.ParallelWaveganGenerator(num_res_blocks=4, stacks=2),
         "univnet": lambda: univnet.UnivnetGenerator(in_channels=64, out_channels=1, hidden_channels=32,
                                                     cond_channels=80, upsample_factors=[8, 8, 4],
                                                     lvc_layers_each_block=4, lvc_kernel_size=3,
                                                     kpnet_hidden_channels=64, kpnet_conv_size=3, dropout=0.0)}[kind]()
    m.eval().to(DEV)
    return lambda b, t=13: m(torch.randn(b, 80, t, device=DEV))


def wavegrad():
    from tts_b200 import wavegrad as W
    small = dict(in_channels=16, y_conv_channels=8, x_conv_channels=32, dblock_out_channels=[16, 16],
                 ublock_out_channels=[32, 16, 16], upsample_factors=[3, 2, 2], upsample_dilations=[[1, 2, 1, 2]] * 3)
    m = W.Wavegrad(W.WavegradConfig(model_params=W.WavegradArgs(**small))).eval().to(DEV)
    m.compute_noise_level(np.linspace(1e-6, 0.01, 3))
    return lambda b, t=13: m.inference(torch.randn(b, 16, t, device=DEV))


def griffin_lim():
    from test_griffin_lim_gpu import ap_for
    from tts_b200.audio import AudioProcessor
    ap = AudioProcessor(verbose=False, **ap_for("1024/256/1024", 3))

    def call(b, t=23):
        lens = torch.tensor([t, t - 6, 3][:b])
        return ap.inv_melspectrogram(torch.rand(b, 80, t, device=DEV) * 8 - 4, lengths=lens)
    return call


CALLS = {
    "hifigan": lambda: hifigan(), "hifigan_window": lambda: hifigan(window=True),
    "flow_reverse": lambda: flow(True), "flow_forward": lambda: flow(False),
    "text_encoder": text_encoder, "sdp": sdp, "posterior": posterior, "duration_predictor": duration_predictor,
    "speaker_encoder": lambda: speaker_encoder(), "speaker_encoder_features": lambda: speaker_encoder(stage=2),
    "glow_tts": lambda: tts("glow_tts"), "forward_tts": lambda: tts("forward_tts"), "overflow": lambda: tts("overflow"),
    "tacotron2": lambda: tts("tacotron2"), "tacotron": lambda: tts("tacotron"),
    "melgan": lambda: vocoder("melgan"), "multiband_melgan": lambda: vocoder("multiband_melgan"),
    "pwgan": lambda: vocoder("pwgan"), "univnet": lambda: vocoder("univnet"), "wavegrad": wavegrad,
    "griffin_lim": griffin_lim,
}


def tensors(out):
    if torch.is_tensor(out):
        return [out]
    if isinstance(out, dict):
        out = out.values()
    return [t for o in out for t in tensors(o)] if isinstance(out, (list, tuple, type({}.values()))) else []


class FakeWorkspace:
    """_lib.workspace handing out exactly `nbytes + short` bytes (short = 0 or -1) followed by a 0xA5 tail; the same
    buffer again for a repeated (tag, size), as the real one does."""

    def __init__(self, short):
        self.short, self.bufs = short, {}

    def __call__(self, device, nbytes, tag="default"):
        n = int(nbytes) + self.short
        if (tag, n) not in self.bufs:
            self.bufs[(tag, n)] = torch.full((n + TAIL,), 0xA5, dtype=torch.uint8, device=device)
        return self.bufs[(tag, n)][:n]

    def tails_intact(self):
        return all(bool((b[-TAIL:] == 0xA5).all()) for b in self.bufs.values())


def seeded(call, b):
    torch.manual_seed(0)
    np.random.seed(0)
    return [t.clone() for t in tensors(call(b))]


@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("name", list(CALLS))
def test_exact_workspace_suffices_and_one_byte_less_is_refused(name, b, monkeypatch):
    call = CALLS[name]()
    want = seeded(call, b)
    fake = FakeWorkspace(0)
    monkeypatch.setattr(_lib, "workspace", fake)
    got = seeded(call, b)
    assert len(got) == len(want) and all(torch.equal(g, w) for g, w in zip(got, want))
    torch.cuda.synchronize()
    assert fake.bufs and fake.tails_intact()
    monkeypatch.setattr(_lib, "workspace", FakeWorkspace(-1))
    before = _lib.launch_count()
    with pytest.raises(RuntimeError, match="workspace"):
        seeded(call, b)
    assert _lib.launch_count() == before


def round256(n):
    return (n + 255) // 256 * 256


def run_raw(fn, nbytes):
    """fn(ws, size) on a buffer of nbytes followed by the 0xA5 tail: its return code and whether the tail is intact."""
    buf = torch.full((nbytes + TAIL,), 0xA5, dtype=torch.uint8, device=DEV)
    rc = fn(_lib.ptr(buf), ctypes.c_size_t(nbytes))
    torch.cuda.synchronize()
    return rc, bool((buf[nbytes:] == 0xA5).all())


@pytest.mark.parametrize("b", [1, 3])
def test_pwgan_layer_workspace(b):
    from tts_b200.pwgan import ParallelWaveganGenerator
    m = ParallelWaveganGenerator(num_res_blocks=4, stacks=2).eval()
    h, L = m._ensure_handle(DEV), _lib.lib()
    t, pad = 13, 2
    tf = t + 2 * pad
    ts = tf * 4 ** 4   # the default upsample_factors [4, 4, 4, 4]
    pitch = (ts + 3) // 4 * 4
    mel = torch.randn(b, 80, t, device=DEV)
    x = torch.randn(b, 64, pitch, device=DEV)
    skip, x_new = torch.zeros_like(x), torch.zeros_like(x)
    st = _lib.stream_ptr(DEV)
    fn = lambda ws, n: L.b200tts_pwgan_layer(h, 1, _lib.ptr(mel), b, t, pad, _lib.ptr(x), _lib.ptr(skip),  # noqa: E731
                                             _lib.ptr(x_new), pitch, ws, n, st)
    need = round256(b * 128 * tf * 4)   # the conditioning of one layer
    assert run_raw(fn, L.b200tts_pwgan_workspace_bytes(h, b, tf)) == (0, True)
    want = x_new.clone()
    assert run_raw(fn, need) == (0, True) and torch.equal(x_new, want)
    before = _lib.launch_count()
    rc, _ = run_raw(fn, need - 1)
    assert rc != 0 and "workspace" in L.b200tts_last_error().decode() and _lib.launch_count() == before


@pytest.mark.parametrize("b", [1, 3])
def test_univnet_predict_workspace(b):
    from tts_b200.univnet import UnivnetGenerator
    m = UnivnetGenerator(in_channels=64, out_channels=1, hidden_channels=32, cond_channels=80, upsample_factors=[8, 8, 4],
                         lvc_layers_each_block=4, lvc_kernel_size=3, kpnet_hidden_channels=64, kpnet_conv_size=3,
                         dropout=0.0).eval()
    h, L = m._ensure_handle(DEV), _lib.lib()
    t = 13
    mel = torch.randn(b, 80, t, device=DEV)
    pred = torch.zeros(b * t * 4 * (6144 + 64), device=DEV)
    st = _lib.stream_ptr(DEV)
    fn = lambda ws, n: L.b200tts_univnet_predict(h, 1, _lib.ptr(mel), b, t, _lib.ptr(pred), ws, n, st)  # noqa: E731
    need = 3 * round256(b * 64 * ((t + 3) // 4 * 4) * 4)   # the kernel predictor's three hidden tensors
    assert run_raw(fn, L.b200tts_univnet_workspace_bytes(h, b, t)) == (0, True)
    want = pred.clone()
    assert run_raw(fn, need) == (0, True) and torch.equal(pred, want)
    before = _lib.launch_count()
    rc, _ = run_raw(fn, need - 1)
    assert rc != 0 and "workspace" in L.b200tts_last_error().decode() and _lib.launch_count() == before
