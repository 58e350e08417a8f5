"""Every engine handle gives back exactly the device buffers it took.

Each handle the library offers is built through its Python module at a small size and dropped again, twice.
b200tts_debug_device_buffers() counts the live device buffers of all handles, so it must rise with the build and come
back to its earlier value with the drop: a buffer a handle leaks, or frees twice, shows up as a difference.
"""
import gc

import pytest
import torch

from tts_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def live_buffers():
    return _lib.lib().b200tts_debug_device_buffers()


def engine(m):
    """EngineModule: handle(device) / _drop_handle()."""
    return lambda: m.handle(DEV), m._drop_handle


def vocoder(m):
    """The vocoders and the speaker encoder: _ensure_handle(device) / _drop_handle()."""
    return lambda: m._ensure_handle(DEV), m._drop_handle


def hifigan():
    from tts_b200.hifigan import HifiganGenerator
    return vocoder(HifiganGenerator(in_channels=20, out_channels=1, resblock_type="1",
                                    resblock_dilation_sizes=[[1, 3, 5]] * 3, resblock_kernel_sizes=[3, 7, 11],
                                    upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=64,
                                    upsample_factors=[8, 8, 2, 2], cond_channels=8).eval())


def flow_reverse():
    from tts_b200.layers import ResidualCouplingBlocks
    m = ResidualCouplingBlocks(8, 16, 5, 1, 2, num_flows=2, cond_channels=4).eval()
    return lambda: m.handle(DEV), m._drop_reverse_handle


def flow_forward():
    from tts_b200.layers import ResidualCouplingBlocks
    m = ResidualCouplingBlocks(8, 16, 5, 1, 2, num_flows=2, cond_channels=4).eval()
    return lambda: m._forward_handle(DEV), m._drop_forward_handle


def text_encoder():
    from tts_b200.layers import TextEncoder
    return engine(TextEncoder(30, 8, 16, 32, 2, 2, 3, 0.1).eval())


def sdp():
    from tts_b200.layers import StochasticDurationPredictor
    return engine(StochasticDurationPredictor(16, 16, 3, 0.5, 4, cond_channels=4).eval())


def posterior():
    from tts_b200.layers import PosteriorEncoder
    return engine(PosteriorEncoder(20, 8, 16, 5, 1, 4, cond_channels=4).eval())


def duration_predictor():
    from tts_b200.layers import DurationPredictor
    return engine(DurationPredictor(16, 32, 3, 0.5, cond_channels=4).eval())


def speaker_encoder():
    from tts_b200.encoder import ResNetSpeakerEncoder
    audio = dict(fft_size=512, win_length=400, hop_length=160, sample_rate=16000, preemphasis=0.97, num_mels=64)
    return vocoder(ResNetSpeakerEncoder(encoder_type="ASP", log_input=True, use_torch_spec=True,
                                        audio_config=audio).eval())


def glow_tts():
    from tts_b200.glow_tts import GlowTTS, GlowTTSConfig
    return engine(GlowTTS(GlowTTSConfig(num_chars=30)).eval())


def forward_tts():
    from tts_b200.forward_tts import FastPitchConfig, ForwardTTS, ForwardTTSArgs
    return engine(ForwardTTS(FastPitchConfig(model_args=ForwardTTSArgs(num_chars=30))).eval())


def melgan():
    from tts_b200.melgan import MelganGenerator
    return vocoder(MelganGenerator(base_channels=64, num_res_blocks=2).eval())


def multiband_melgan():   # with the PQMF synthesis filter
    from tts_b200.melgan import MultibandMelganGenerator
    return vocoder(MultibandMelganGenerator(base_channels=64, num_res_blocks=2).eval())


def fullband_melgan():
    from tts_b200.melgan import FullbandMelganGenerator
    return vocoder(FullbandMelganGenerator(base_channels=64, num_res_blocks=2).eval())


def wavegrad():
    from tts_b200 import wavegrad as W
    small = dict(in_channels=16, y_conv_channels=8, x_conv_channels=32, dblock_out_channels=[16, 16],
                 ublock_out_channels=[32, 16, 16], upsample_factors=[3, 2, 2], upsample_dilations=[[1, 2, 1, 2]] * 3)
    return vocoder(W.Wavegrad(W.WavegradConfig(model_params=W.WavegradArgs(**small))).eval())


def pwgan():
    from tts_b200.pwgan import ParallelWaveganGenerator
    return vocoder(ParallelWaveganGenerator(num_res_blocks=4, stacks=2).eval())


def univnet():
    from tts_b200.univnet import UnivnetGenerator
    return vocoder(UnivnetGenerator(in_channels=64, out_channels=1, hidden_channels=32, cond_channels=80,
                                    upsample_factors=[8, 8, 4], lvc_layers_each_block=4, lvc_kernel_size=3,
                                    kpnet_hidden_channels=64, kpnet_conv_size=3, dropout=0.0).eval())


def overflow():   # with the Glow decoder
    from tts_b200 import overflow as OV
    return engine(OV.Overflow(OV.OverflowConfig(num_chars=30)).eval())


def tacotron2():
    from tts_b200 import tacotron2 as TC
    return engine(TC.Tacotron2(TC.Tacotron2Config(num_chars=30)).eval())


def fused_conv1d():   # split-fp16 at 64 rows: plain and grouped tensor-core images and their row scales
    from tts_b200.conv import FusedConv1d
    conv = FusedConv1d(torch.randn(64, 64, 3) * 0.1, torch.randn(64), padding=1, precision="f16x3")

    def drop():
        for h in conv._handles.values():
            _lib.lib().b200tts_conv1d_destroy(h)
        conv._handles.clear()
    return lambda: conv._handle(DEV), drop


def stft():   # with the mel projection
    from tts_b200 import audio
    basis = audio.mel_filterbank(8000, 64, 10)
    cached = set(audio._handles)

    def build():
        audio._handle(DEV, 64, 7, 48, "hann_window", mel_key="test_device_buffers", mel_basis=basis)

    def drop():
        for key in set(audio._handles) - cached:
            _lib.lib().b200tts_stft_destroy(audio._handles.pop(key))
    return build, drop


HANDLES = [hifigan, flow_reverse, flow_forward, text_encoder, sdp, posterior, duration_predictor, speaker_encoder,
           glow_tts, forward_tts, melgan, multiband_melgan, fullband_melgan, wavegrad, pwgan, univnet, overflow,
           tacotron2, fused_conv1d, stft]


@pytest.mark.parametrize("make", HANDLES, ids=[f.__name__ for f in HANDLES])
def test_handle_frees_every_device_buffer_it_made(make):
    torch.manual_seed(0)
    build, drop = make()
    # handles of earlier tests that only a garbage collection frees must not be freed during build(): the count would
    # drop by theirs
    gc.collect()
    before = live_buffers()
    for _ in range(2):
        build()
        torch.cuda.synchronize()
        assert live_buffers() > before, "building the handle made no device buffer"
        drop()
        assert live_buffers() == before, f"{live_buffers() - before:+d} device buffers after dropping the handle"
