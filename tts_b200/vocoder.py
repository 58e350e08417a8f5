"""The standalone-vocoder side of the path: config / model discovery and the hand-off around the HiFiGAN generator.

Mirrors, with the reference's names and argument meaning:
  HifiganConfig        <- /root/reference/TTS/vocoder/configs/hifigan_config.py:7-136 (+ BaseAudioConfig,
                          TTS/config/shared_configs.py:9-176: the audio fields the hand-off reads)
  MelganConfig / MultibandMelganConfig / FullbandMelganConfig
                       <- TTS/vocoder/configs/{melgan,multiband_melgan,fullband_melgan}_config.py (generator side)
  setup_generator(c)   <- TTS/vocoder/models/__init__.py:34-94   (the HiFiGAN and MelGAN generator families)
  GAN                  <- TTS/vocoder/models/gan.py:21-66,338-352 (model_g, forward, inference, load_checkpoint)
  AudioProcessor.normalize / denormalize   <- TTS/utils/audio/processor.py:259-337   (as ``AudioNorm``)
  interpolate_vocoder_input                <- TTS/vocoder/utils/generic_utils.py:11-29
  vocoder_input(...)   <- the chain of TTS/utils/synthesizer.py:412-429 + the replicate pad of
                          HifiganGenerator.inference (hifigan_generator.py:281) in ONE device pass
  wav_to_int16         <- save_wav's peak normalisation, TTS/utils/audio/numpy_transforms.py:439-441

Everything numeric runs in libtts_b200.so (``b200tts_vocoder_input`` / ``b200tts_absmax`` / ``b200tts_to_int16``).
"""
import ctypes
import math
from dataclasses import dataclass, field
from typing import Optional

import torch
from torch import nn

from . import _lib
from .hifigan import HifiganGenerator
from .melgan import FullbandMelganGenerator, MelganGenerator, MultibandMelganGenerator


# ----------------------------------------------------------------------------- configs
class _ItemAccess:
    def __getitem__(self, k):
        return getattr(self, k)

    def __setitem__(self, k, v):
        setattr(self, k, v)

    def __contains__(self, k):
        return hasattr(self, k)

    def get(self, k, default=None):
        return getattr(self, k, default)


@dataclass
class BaseAudioConfig(_ItemAccess):
    """The fields of TTS/config/shared_configs.py:9-176 that the vocoder hand-off reads (same names and defaults)."""
    fft_size: int = 1024
    win_length: int = 1024
    hop_length: int = 256
    sample_rate: int = 22050
    num_mels: int = 80
    mel_fmin: float = 0.0
    mel_fmax: float = None
    ref_level_db: int = 20
    min_level_db: int = -100
    signal_norm: bool = True
    symmetric_norm: bool = True
    max_norm: float = 4.0
    clip_norm: bool = True
    stats_path: str = None


@dataclass
class HifiganConfig(_ItemAccess):
    """Generator-side fields of TTS/vocoder/configs/hifigan_config.py:91-104 (the loss / discriminator / trainer
    fields of the training recipe are out of scope)."""
    model: str = "hifigan"
    discriminator_model: str = "hifigan_discriminator"
    generator_model: str = "hifigan_generator"
    generator_model_params: dict = field(default_factory=lambda: {
        "upsample_factors": [8, 8, 2, 2],
        "upsample_kernel_sizes": [16, 16, 4, 4],
        "upsample_initial_channel": 512,
        "resblock_kernel_sizes": [3, 7, 11],
        "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
        "resblock_type": "1",
    })
    audio: BaseAudioConfig = field(default_factory=BaseAudioConfig)


_MELGAN_DISCRIMINATOR = "melgan_multiscale_discriminator"


@dataclass
class MelganConfig(_ItemAccess):
    """Generator-side fields of TTS/vocoder/configs/melgan_config.py:65-75 (+ ``use_pqmf`` of the shared GAN config)."""
    model: str = "melgan"
    discriminator_model: str = _MELGAN_DISCRIMINATOR
    generator_model: str = "melgan_generator"
    generator_model_params: dict = field(default_factory=lambda: {"upsample_factors": [8, 8, 2, 2], "num_res_blocks": 3})
    use_pqmf: bool = False
    audio: BaseAudioConfig = field(default_factory=BaseAudioConfig)


@dataclass
class MultibandMelganConfig(_ItemAccess):
    """Generator-side fields of TTS/vocoder/configs/multiband_melgan_config.py:93-102."""
    model: str = "multiband_melgan"
    discriminator_model: str = _MELGAN_DISCRIMINATOR
    generator_model: str = "multiband_melgan_generator"
    generator_model_params: dict = field(default_factory=lambda: {"upsample_factors": [8, 4, 2], "num_res_blocks": 4})
    use_pqmf: bool = True
    audio: BaseAudioConfig = field(default_factory=BaseAudioConfig)


@dataclass
class FullbandMelganConfig(_ItemAccess):
    """Generator-side fields of TTS/vocoder/configs/fullband_melgan_config.py:65-75.  As in the reference, the generator
    it names is ``melgan_generator`` (a plain MelGAN with 4 residual blocks), not ``fullband_melgan_generator``."""
    model: str = "fullband_melgan"
    discriminator_model: str = _MELGAN_DISCRIMINATOR
    generator_model: str = "melgan_generator"
    generator_model_params: dict = field(default_factory=lambda: {"upsample_factors": [8, 8, 2, 2], "num_res_blocks": 4})
    use_pqmf: bool = False
    audio: BaseAudioConfig = field(default_factory=BaseAudioConfig)


# the generator modules under TTS/vocoder/models/ that setup_generator can import
_GENERATOR_MODULES = ("hifigan_generator", "melgan_generator", "multiband_melgan_generator", "fullband_melgan_generator",
                      "parallel_wavegan_generator", "univnet_generator")


class GeneratorParamsError(KeyError, NotImplementedError):
    """``generator_model_params`` lacks a field the named generator needs (the reference raises KeyError there); also a
    NotImplementedError, so that callers that treat an unbuildable generator as such keep working."""


def to_camel(text):
    """TTS/vocoder/models/__init__.py:7-9 (generator_model name -> class name)."""
    text = text.capitalize()
    return "".join(ch.upper() if i and text[i - 1] == "_" else ch for i, ch in enumerate(text) if ch != "_")


def setup_generator(c):
    """TTS/vocoder/models/__init__.py:34-94: builds the generator a vocoder config names, resolving the name the way the
    reference does.  The reference first imports the module ``TTS.vocoder.models.<name.lower()>``, so only the names of
    its generator modules (in any letter case) get as far as its ``name in "..."`` substring tests; any other name
    raises NotImplementedError here (the reference fails it at that import).  ``melgan_fb_generator`` raises the
    reference's ValueError ("now fullband_melgan_generator").  The HiFiGAN and MelGAN families are on the path;
    ParallelWaveGAN and UniVNet are out of scope and raise NotImplementedError."""
    name = _get(c, "generator_model")
    low = name.lower()
    if name == "melgan_fb_generator":
        raise ValueError("melgan_fb_generator is now fullband_melgan_generator")
    if low not in _GENERATOR_MODULES:
        raise NotImplementedError(f"tts_b200.setup_generator: `{name}` names no generator module "
                                  f"(one of {sorted(_GENERATOR_MODULES)})")
    num_mels = _get(_get(c, "audio"), "num_mels")
    params = _get(c, "generator_model_params")

    def param(key):
        try:
            return params[key]
        except KeyError:
            raise GeneratorParamsError(f"tts_b200.setup_generator: `{name}` needs generator_model_params[{key!r}]") from None

    if low in "hifigan_generator":
        return HifiganGenerator(in_channels=num_mels, out_channels=1, **dict(params))
    melgan = dict(proj_kernel=7, res_kernel=3)
    if low in "melgan_generator":
        return MelganGenerator(in_channels=num_mels, out_channels=1, base_channels=512,
                               upsample_factors=param("upsample_factors"), num_res_blocks=param("num_res_blocks"), **melgan)
    if low in "multiband_melgan_generator":
        return MultibandMelganGenerator(in_channels=num_mels, out_channels=4, base_channels=384,
                                        upsample_factors=param("upsample_factors"), num_res_blocks=param("num_res_blocks"),
                                        **melgan)
    if low in "fullband_melgan_generator":
        return FullbandMelganGenerator(in_channels=num_mels, out_channels=1, base_channels=512,
                                       upsample_factors=param("upsample_factors"), num_res_blocks=param("num_res_blocks"),
                                       **melgan)
    raise NotImplementedError(f"tts_b200.setup_generator: `{name}` is not built (the HiFiGAN and MelGAN generators are)")


def setup_model(config):
    """TTS/vocoder/models/__init__.py:12-31: ``GAN`` for a config naming both a generator and a discriminator or for
    ``model == "gan"`` (then built by ``setup_generator`` from ``generator_model``, as the reference's GAN does),
    ``Wavegrad`` for ``model == "wavegrad"``.  The other vocoder models that function can name (WaveRNN, ...) are not
    built here and raise NotImplementedError, as does a config without a ``model`` name."""
    if "discriminator_model" in config and "generator_model" in config:
        return GAN.init_from_config(config)
    model = _get(config, "model")
    if not isinstance(model, str):
        raise NotImplementedError("tts_b200.setup_model: the config names no vocoder `model` (and no generator + "
                                  "discriminator pair)")
    name = model.lower()
    if name == "gan":
        return GAN.init_from_config(config)
    if name == "wavegrad":
        from .wavegrad import Wavegrad   # wavegrad.py imports this module's config classes
        return Wavegrad.init_from_config(config)
    raise NotImplementedError(f"tts_b200.setup_model: vocoder model `{_get(config, 'model')}` is not built "
                              "(GAN generators and WaveGrad are)")


def _get(obj, key, default=None):
    if isinstance(obj, dict):
        return obj.get(key, default)
    return getattr(obj, key, default)


class GAN(nn.Module):
    """Inference surface of TTS/vocoder/models/gan.py: ``model_g`` built by ``setup_generator``; ``forward`` /
    ``inference`` delegate to it (gan.py:46-66); ``load_checkpoint`` as gan.py:338-352 (accepts both the trainer
    checkpoint with ``model_g.*`` keys and the bare-generator checkpoints older zoo vocoders ship)."""

    def __init__(self, config, ap=None):
        super().__init__()
        self.config = config
        self.ap = ap
        self.model_g = setup_generator(config)
        self.model_d = None          # the discriminator is training-only

    def forward(self, x):
        return self.model_g.forward(x)

    def inference(self, x):
        return self.model_g.inference(x)

    def load_checkpoint(self, config, checkpoint_path, eval=False, cache=False):  # pylint: disable=redefined-builtin
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        if "model_disc" in state:            # old-format generator-only checkpoint (gan.py:343-345)
            self.model_g.load_checkpoint(config, checkpoint_path, eval)
        else:
            model = {k: v for k, v in state["model"].items() if not k.startswith("model_d.")}
            self.load_state_dict(model, strict=True)
            if eval:
                self.model_d = None
                if hasattr(self.model_g, "remove_weight_norm"):
                    self.model_g.remove_weight_norm()
                self.eval()

    @staticmethod
    def init_from_config(config, verbose=True):
        return GAN(config)


# ----------------------------------------------------------------------------- AudioProcessor normalisation
@dataclass
class AudioNorm:
    """The normalisation state of one ``AudioProcessor`` (processor.py:140-230): range normalisation
    (``ref_level_db`` / ``min_level_db`` / ``max_norm``, symmetric or not, clipped or not) or the mean-var scaler of a
    ``stats_path`` (``mel_mean`` / ``mel_std`` as the ``StandardScaler`` holds them)."""
    signal_norm: bool = True
    symmetric_norm: bool = True
    max_norm: float = 4.0
    clip_norm: bool = True
    min_level_db: float = -100.0
    ref_level_db: float = 20.0
    mel_mean: Optional[torch.Tensor] = None
    mel_std: Optional[torch.Tensor] = None

    @staticmethod
    def from_audio_config(audio):
        """From an audio config (dict / dataclass with the AudioProcessor constructor's field names); ``None``
        values take the constructor's fallbacks (processor.py:176-199: ``min_level_db or 0``, ``max_norm`` 1.0 ...)."""
        g = lambda k, d=None: _get(audio, k, d)
        mx = g("max_norm")
        return AudioNorm(signal_norm=bool(g("signal_norm")), symmetric_norm=bool(g("symmetric_norm")),
                         max_norm=1.0 if mx is None else float(mx), clip_norm=bool(g("clip_norm", True)),
                         min_level_db=float(g("min_level_db") or 0), ref_level_db=float(g("ref_level_db") or 0))

    @staticmethod
    def identity():
        return AudioNorm(signal_norm=False)

    def _c(self, device, keep):
        s = _lib.AudioNormC()
        s.signal_norm, s.symmetric_norm, s.clip_norm = int(self.signal_norm), int(self.symmetric_norm), int(self.clip_norm)
        s.max_norm, s.min_level_db, s.ref_level_db = float(self.max_norm), float(self.min_level_db), float(self.ref_level_db)
        if self.signal_norm and self.mel_mean is not None:
            mean = torch.as_tensor(self.mel_mean, dtype=torch.float32).to(device).contiguous()
            std = torch.as_tensor(self.mel_std, dtype=torch.float32).to(device).contiguous()
            keep += [mean, std]
            s.scaler_mean, s.scaler_scale = mean.data_ptr(), std.data_ptr()
        return s

    def normalize(self, S):
        """``AudioProcessor.normalize`` (processor.py:259-301) on a CUDA spectrogram [C,T] or [B,C,T]."""
        return vocoder_input(S, AudioNorm.identity(), self)

    def denormalize(self, S):
        """``AudioProcessor.denormalize`` (processor.py:303-337)."""
        return vocoder_input(S, self, AudioNorm.identity())


def vocoder_input(spec, tts_norm, vocoder_norm, scale_factor=1.0, padding=0, time_last=True, aligned=False):
    """``vocoder_norm.normalize(tts_norm.denormalize(spec))`` -> bilinear interpolation along time by ``scale_factor``
    -> ``padding`` replicated frames each side, in one kernel.  spec: CUDA [C,T] / [B,C,T] (``time_last``) or the TTS
    model's [B,T,C] output (``time_last=False``).  Returns [B,C,T'] (or [C,T'] for 2-D input); ``aligned=True`` returns
    a view with a 16-byte aligned row pitch (what the tensor-core kernels want)."""
    _lib.require_cuda(spec, "spec")
    squeeze = spec.dim() == 2
    x = spec.unsqueeze(0) if squeeze else spec
    x = x.to(torch.float32)
    if time_last:
        b, c, t = x.shape
        sb, sc, st = x.stride()
    else:
        b, t, c = x.shape
        sb, st, sc = x.stride()
    L = _lib.lib()
    tout = L.b200tts_vocoder_input_len(t, ctypes.c_float(scale_factor), int(padding))
    pitch = (tout + 3) // 4 * 4 if aligned else tout
    y = torch.empty((b, c, pitch), dtype=torch.float32, device=x.device)
    keep = []
    dn, nm = tts_norm._c(x.device, keep), vocoder_norm._c(x.device, keep)
    with torch.cuda.device(x.device):
        rc = L.b200tts_vocoder_input(_lib.ptr(x), ctypes.c_longlong(sb), int(sc), int(st), b, c, t, ctypes.byref(dn),
                                     ctypes.byref(nm), ctypes.c_float(scale_factor), int(padding), _lib.ptr(y), pitch,
                                     _lib.stream_ptr(x.device))
    _lib.check(rc, "vocoder_input")
    y = y[:, :, :tout]
    return y[0] if squeeze else y


def interpolate_vocoder_input(scale_factor, spec):
    """TTS/vocoder/utils/generic_utils.py:11-29: spec [C,T] -> [1,C,floor(T*scale_factor[1])] (bilinear,
    align_corners=False, recompute_scale_factor=True).  ``scale_factor`` is the reference's ``[1, r]`` pair."""
    r = float(scale_factor[1]) if isinstance(scale_factor, (list, tuple)) else float(scale_factor)
    if isinstance(scale_factor, (list, tuple)) and float(scale_factor[0]) != 1.0:
        raise NotImplementedError("tts_b200.interpolate_vocoder_input: the reference only scales the time axis")
    spec = torch.as_tensor(spec)
    return vocoder_input(spec, AudioNorm.identity(), AudioNorm.identity(), scale_factor=r).unsqueeze(0)


# ----------------------------------------------------------------------------- save_wav's peak normalisation
def new_peak(device):
    """A zeroed device word for ``HifiganGenerator.forward(..., peak=...)`` / ``wav_to_int16(..., peak=...)``."""
    return torch.zeros(1, dtype=torch.int32, device=device)


def wav_to_int16(wav, peak=None):
    """``(wav * (32767 / max(0.01, max|wav|))).astype(int16)`` (numpy_transforms.py:439-441) on the device.  ``peak``:
    the word conv_post already folded max|wav| into (``waveform_decoder(z, peak=p)``); computed here when None."""
    _lib.require_cuda(wav, "wav")
    wav = wav.to(torch.float32).contiguous()
    out = torch.empty(wav.shape, dtype=torch.int16, device=wav.device)
    L = _lib.lib()
    with torch.cuda.device(wav.device):
        if peak is None:
            peak = new_peak(wav.device)
            _lib.check(L.b200tts_absmax(_lib.ptr(wav), ctypes.c_longlong(wav.numel()), _lib.ptr(peak),
                                        _lib.stream_ptr(wav.device)), "absmax")
        _lib.check(L.b200tts_to_int16(_lib.ptr(wav), ctypes.c_longlong(wav.numel()), _lib.ptr(peak), _lib.ptr(out),
                                      _lib.stream_ptr(wav.device)), "to_int16")
    return out
