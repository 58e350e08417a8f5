"""Drop-in for the WaveGrad vocoder of the reference:

  WavegradArgs / WavegradConfig  <- TTS/vocoder/models/wavegrad.py:20-31, TTS/vocoder/configs/wavegrad_config.py:8-90
                                    (the model-side fields, both noise schedules and ``audio``)
  Wavegrad                       <- TTS/vocoder/models/wavegrad.py:34-245 (inference surface), with the layers of
                                    TTS/vocoder/layers/wavegrad.py:19-154 as parameter containers

Same constructor, same ``state_dict`` keys with and without weight norm (legacy ``weight_g`` / ``weight_v`` checkpoints
load through torch's weight-norm compatibility hook), same ``forward(x, spectrogram, noise_scale)``, ``inference``,
``compute_noise_level``, ``load_noise_schedule``, ``load_checkpoint`` and weight-norm helpers.  The arithmetic runs in
libtts_b200.so (``b200tts_wavegrad_*``); there is no PyTorch fallback.

``inference(x, y_n=None, *, init_noise=None, step_noise=None)`` draws its noise exactly as the reference does -- the
initial signal ``torch.randn(B, 1, hop * T)`` on the CPU generator, then one ``torch.randn_like(y)`` on the device
generator after every step n > 0 -- so under the same seeds it consumes the same random numbers.  ``init_noise`` [B, 1, L]
and ``step_noise`` [N - 1, B, 1, L] (``step_noise[n - 1]`` is the z of step n, the one ``sigma[n - 1]`` scales) replace
those draws.  The spectrogram's ``x_conv`` runs once per call, and each of the N steps is one engine call with no host
synchronisation.
"""
import ctypes
from dataclasses import dataclass, field
from typing import List

import numpy as np
import torch
from torch import nn
from torch.nn.utils.parametrizations import weight_norm
from torch.nn.utils.parametrize import is_parametrized, remove_parametrizations

from . import _lib
from .vocoder import BaseAudioConfig, _ItemAccess


@dataclass
class WavegradArgs(_ItemAccess):
    """TTS/vocoder/models/wavegrad.py:20-31."""
    in_channels: int = 80
    out_channels: int = 1
    use_weight_norm: bool = False
    y_conv_channels: int = 32
    x_conv_channels: int = 768
    dblock_out_channels: List[int] = field(default_factory=lambda: [128, 128, 256, 512])
    ublock_out_channels: List[int] = field(default_factory=lambda: [512, 512, 256, 128, 128])
    upsample_factors: List[int] = field(default_factory=lambda: [4, 4, 4, 2, 2])
    upsample_dilations: List[List[int]] = field(
        default_factory=lambda: [[1, 2, 1, 2], [1, 2, 1, 2], [1, 2, 4, 8], [1, 2, 4, 8], [1, 2, 4, 8]])


@dataclass
class WavegradConfig(_ItemAccess):
    """Model-side fields of TTS/vocoder/configs/wavegrad_config.py:73-90 (the training recipe's optimiser fields are out
    of scope).  It names no discriminator, so ``setup_model`` builds ``Wavegrad``."""
    model: str = "wavegrad"
    generator_model: str = "wavegrad"
    model_params: WavegradArgs = field(default_factory=WavegradArgs)
    train_noise_schedule: dict = field(default_factory=lambda: {"min_val": 1e-6, "max_val": 1e-2, "num_steps": 1000})
    test_noise_schedule: dict = field(default_factory=lambda: {"min_val": 1e-6, "max_val": 1e-2, "num_steps": 50})
    audio: BaseAudioConfig = field(default_factory=BaseAudioConfig)


def _conv(cin, cout, k, dilation=1, padding=0):
    return nn.Conv1d(cin, cout, k, dilation=dilation, padding=padding)


class _FiLM(nn.Module):
    """layers/wavegrad.py:40-63: ``input_conv`` / ``output_conv`` (the PositionalEncoding holds no state-dict entry)."""

    def __init__(self, input_size, output_size):
        super().__init__()
        self.input_conv = _conv(input_size, input_size, 3, padding=1)
        self.output_conv = _conv(input_size, output_size * 2, 3, padding=1)

    def apply_weight_norm(self):
        self.input_conv = weight_norm(self.input_conv)
        self.output_conv = weight_norm(self.output_conv)


class _UBlock(nn.Module):
    """layers/wavegrad.py:74-123."""

    def __init__(self, input_size, hidden_size, factor, dilation):
        super().__init__()
        assert isinstance(dilation, (list, tuple))
        assert len(dilation) == 4
        self.factor = factor
        self.res_block = _conv(input_size, hidden_size, 1)
        self.main_block = nn.ModuleList([_conv(input_size, hidden_size, 3, dilation[0], dilation[0]),
                                         _conv(hidden_size, hidden_size, 3, dilation[1], dilation[1])])
        self.out_block = nn.ModuleList([_conv(hidden_size, hidden_size, 3, dilation[2], dilation[2]),
                                        _conv(hidden_size, hidden_size, 3, dilation[3], dilation[3])])

    def apply_weight_norm(self):
        self.res_block = weight_norm(self.res_block)
        for blocks in (self.main_block, self.out_block):
            for i, layer in enumerate(blocks):
                blocks[i] = weight_norm(layer)


class _DBlock(nn.Module):
    """layers/wavegrad.py:133-163."""

    def __init__(self, input_size, hidden_size, factor):
        super().__init__()
        self.factor = factor
        self.res_block = _conv(input_size, hidden_size, 1)
        self.main_block = nn.ModuleList([_conv(input_size, hidden_size, 3, 1, 1), _conv(hidden_size, hidden_size, 3, 2, 2),
                                         _conv(hidden_size, hidden_size, 3, 4, 4)])

    def apply_weight_norm(self):
        self.res_block = weight_norm(self.res_block)
        for i, layer in enumerate(self.main_block):
            self.main_block[i] = weight_norm(layer)


def _pe_table(n_channels, length):
    """PositionalEncoding.init_pe_matrix (layers/wavegrad.py:30-37) over ``length`` positions, divided by C = 5000 as its
    forward does -- the same CPU float32 operations, so the same values."""
    pe = torch.zeros(length, n_channels)
    position = torch.arange(0, length, dtype=torch.float).unsqueeze(1)
    div_term = torch.pow(10000, torch.arange(0, n_channels, 2).float() / n_channels)
    pe[:, 0::2] = torch.sin(position / div_term)
    pe[:, 1::2] = torch.cos(position / div_term)
    return pe.transpose(0, 1) / 5000


class Wavegrad(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        p = config.model_params
        self.use_weight_norm = p.use_weight_norm
        self.hop_len = int(np.prod(p.upsample_factors))
        self.noise_level = self.num_steps = self.beta = self.alpha = self.alpha_hat = None
        self.c1 = self.c2 = self.sigma = None
        n = len(p.upsample_factors)
        if not (len(p.ublock_out_channels) == n and len(p.upsample_dilations) == n and len(p.dblock_out_channels) == n - 1):
            raise NotImplementedError("tts_b200.Wavegrad: needs len(ublock_out_channels) == len(upsample_dilations) == "
                                      "len(upsample_factors) == len(dblock_out_channels) + 1 (every block and FiLM used)")
        if list(p.dblock_out_channels) != list(reversed(p.ublock_out_channels))[: n - 1]:
            # FiLM i + 1 is built for reversed(ublock_out_channels)[i] input channels and reads DBlock i's output: the
            # reference fails such a config at its first forward with a shape error
            raise ValueError("tts_b200.Wavegrad: dblock_out_channels must equal reversed(ublock_out_channels)[:-1] (FiLM i + 1 "
                             f"reads DBlock i's output), got {list(p.dblock_out_channels)} and {list(p.ublock_out_channels)}")
        self.y_conv = _conv(1, p.y_conv_channels, 5, padding=2)
        self.dblocks = nn.ModuleList()
        ic = p.y_conv_channels
        for oc, df in zip(p.dblock_out_channels, reversed(p.upsample_factors)):
            self.dblocks.append(_DBlock(ic, oc, df))
            ic = oc
        self.film = nn.ModuleList()
        ic = p.y_conv_channels
        for oc in reversed(p.ublock_out_channels):
            self.film.append(_FiLM(ic, oc))
            ic = oc
        self.ublocks = nn.ModuleList()
        ic = p.x_conv_channels
        for oc, uf, ud in zip(p.ublock_out_channels, p.upsample_factors, p.upsample_dilations):
            self.ublocks.append(_UBlock(ic, oc, uf, ud))
            ic = oc
        self.x_conv = _conv(p.in_channels, p.x_conv_channels, 3, padding=1)
        self.out_conv = _conv(oc, p.out_channels, 3, padding=1)
        if p.use_weight_norm:
            self.apply_weight_norm()
        self._handle = None
        self._handle_device = None
        self._pe = None              # (device, frames, tables, pointer array)
        self._register_load_state_dict_pre_hook(lambda *a, **k: self._drop_handle())

    # ------------------------------------------------------------------ engine handle
    def _drop_handle(self):
        if getattr(self, "_handle", None) is not None:
            _lib.lib().b200tts_wavegrad_destroy(self._handle)
        self._handle = None

    def __del__(self):
        try:
            self._drop_handle()
        except Exception:  # pragma: no cover - interpreter shutdown
            pass

    def _apply(self, fn, *a, **kw):
        self._drop_handle()
        return super()._apply(fn, *a, **kw)

    def repack(self):
        """Re-read the parameters (call after modifying weights in place)."""
        self._drop_handle()

    def _convs(self):
        """The convs in state-dict order (the weight order of include/tts_b200.h)."""
        out = [self.y_conv]
        for d in self.dblocks:
            out += [d.res_block, *d.main_block]
        for f in self.film:
            out += [f.input_conv, f.output_conv]
        for u in self.ublocks:
            out += [u.res_block, *u.main_block, *u.out_block]
        return out + [self.x_conv, self.out_conv]

    def _ensure_handle(self, device):
        if self._handle is not None and self._handle_device == device:
            return self._handle
        self._drop_handle()
        p = self.config.model_params
        n = len(p.upsample_factors)
        if not 1 <= n <= 8 or p.out_channels != 1:
            raise NotImplementedError("tts_b200.Wavegrad: 1 to 8 upsample factors and out_channels 1 are supported")
        cfg = _lib.WavegradConfigC()
        cfg.in_channels, cfg.out_channels = p.in_channels, p.out_channels
        cfg.y_conv_channels, cfg.x_conv_channels, cfg.num_upsamples = p.y_conv_channels, p.x_conv_channels, n
        for i in range(n):
            cfg.upsample_factors[i] = p.upsample_factors[i]
            cfg.ublock_out_channels[i] = p.ublock_out_channels[i]
            for k in range(4):
                cfg.upsample_dilations[i][k] = p.upsample_dilations[i][k]
            if i + 1 < n:
                cfg.dblock_out_channels[i] = p.dblock_out_channels[i]
        tensors = []
        with torch.no_grad():
            for m in self._convs():
                tensors += [m.weight.detach().to(torch.float32).cpu().contiguous(),
                            m.bias.detach().to(torch.float32).cpu().contiguous()]
        arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            rc = _lib.lib().b200tts_wavegrad_create(ctypes.byref(cfg), arr, len(tensors), ctypes.byref(handle))
        _lib.check(rc, "wavegrad_create")
        self._handle, self._handle_device = handle, device
        return handle

    def _film_lengths(self, T):
        f = self.config.model_params.upsample_factors
        L = [self.hop_len * T]
        for df in reversed(f[1:]):
            L.append(L[-1] // df)
        return L

    def _pe_tables(self, device, T):
        """Device tables pe / 5000 of every FiLM, one set, rebuilt only when a longer input (or another device) arrives
        -- the reference's cache rule, so memory stays bounded by the longest input.  Returns (pointer array, the frame
        count the tables were built for: their row pitch is each FiLM's length at that count)."""
        if self._pe is None or self._pe[0] != device or self._pe[1] < T:
            self._pe = None                                    # free the old set before building the new one
            p = self.config.model_params
            chans = [p.y_conv_channels] + list(p.dblock_out_channels)   # FiLM i's input channels
            tabs = [_pe_table(c, L).to(device).contiguous() for c, L in zip(chans, self._film_lengths(T))]
            self._pe = (device, T, tabs, (ctypes.c_void_p * len(tabs))(*[t.data_ptr() for t in tabs]))
        return self._pe[3], self._pe[1]

    def _prepare(self, spectrogram):
        dev = self.x_conv.bias.device
        _lib.require_cuda(self.x_conv.bias, "the model's parameters")
        x = spectrogram.to(device=dev, dtype=torch.float32).contiguous()
        if x.dim() != 3 or x.shape[1] != self.config.model_params.in_channels:
            raise ValueError(f"tts_b200.Wavegrad: expected [B, {self.config.model_params.in_channels}, T], got "
                             f"{tuple(x.shape)}")
        return x

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    def forward(self, x, spectrogram, noise_scale):
        """wavegrad.py:106-120: x [B, 1, hop T] (the noisy signal), spectrogram [B, in, T], noise_scale [B] -> the
        network output [B, 1, hop T]."""
        c = self._prepare(spectrogram)
        b, _, t = c.shape
        y = x.to(device=c.device, dtype=torch.float32).contiguous()
        if tuple(y.shape) != (b, 1, self.hop_len * t):
            raise ValueError(f"tts_b200.Wavegrad.forward: x must be [{b}, 1, {self.hop_len * t}], got {tuple(y.shape)}")
        ns = torch.as_tensor(noise_scale, dtype=torch.float32).to(c.device).reshape(-1).expand(b).contiguous()
        h = self._ensure_handle(c.device)
        L = _lib.lib()
        eps = torch.empty_like(y)
        with torch.cuda.device(c.device):
            ws = _lib.workspace(c.device, L.b200tts_wavegrad_workspace_bytes(h, b, t), "wavegrad")
            pe, pe_frames = self._pe_tables(c.device, t)
            rc = L.b200tts_wavegrad_forward(h, _lib.ptr(y), _lib.ptr(c), _lib.ptr(ns), pe, pe_frames, b, t, _lib.ptr(eps),
                                            _lib.ptr(ws), ctypes.c_size_t(ws.numel()), _lib.stream_ptr(c.device))
        _lib.check(rc, "wavegrad_forward")
        return eps

    @torch.no_grad()
    def inference(self, x, y_n=None, *, init_noise=None, step_noise=None):
        """wavegrad.py:126-145: N = len(alpha) refinement steps from noise, conditioned on x [B, in, T] ->
        [B, 1, hop T].  ``y_n`` (a 1-D array, B = 1) is the reference's starting signal; ``init_noise`` /
        ``step_noise`` replace the random draws (see the module docstring)."""
        if self.alpha is None:
            raise RuntimeError("tts_b200.Wavegrad.inference: no noise schedule (compute_noise_level / load_checkpoint)")
        c = self._prepare(x)
        b, _, t = c.shape
        n_steps = len(self.alpha)
        shape = (b, 1, self.hop_len * t)
        if y_n is not None:
            y = torch.FloatTensor(y_n).unsqueeze(0).unsqueeze(0)
            if b != 1 or tuple(y.shape) != shape:
                raise ValueError(f"tts_b200.Wavegrad.inference: y_n must have {shape[2]} samples and B must be 1")
        elif init_noise is not None:
            y = torch.as_tensor(init_noise)
        else:
            y = torch.randn(b, 1, self.hop_len * t)
        y = y.to(device=c.device, dtype=torch.float32).contiguous().clone()
        if tuple(y.shape) != shape:
            raise ValueError(f"tts_b200.Wavegrad.inference: init_noise must be {shape}, got {tuple(y.shape)}")
        if step_noise is not None:
            step_noise = torch.as_tensor(step_noise).to(device=c.device, dtype=torch.float32).contiguous()
            if tuple(step_noise.shape) != (n_steps - 1,) + shape:
                raise ValueError(f"tts_b200.Wavegrad.inference: step_noise must be {(n_steps - 1,) + shape}, got "
                                 f"{tuple(step_noise.shape)}")
        levels = self.noise_level.to(c.device)[:, None].repeat(1, b).contiguous()     # [N, B]: noise_level[n].repeat(B)
        c1, c2, sigma = self.c1.tolist(), self.c2.tolist(), self.sigma.tolist()        # CPU tensors: no device sync
        h = self._ensure_handle(c.device)
        L = _lib.lib()
        with torch.cuda.device(c.device):
            ws = _lib.workspace(c.device, L.b200tts_wavegrad_workspace_bytes(h, b, t), "wavegrad")
            pe, pe_frames = self._pe_tables(c.device, t)
            st = _lib.stream_ptr(c.device)
            _lib.check(L.b200tts_wavegrad_condition(h, _lib.ptr(c), b, t, _lib.ptr(ws), ctypes.c_size_t(ws.numel()), st),
                       "wavegrad_condition")
            for n in range(n_steps - 1, -1, -1):
                z = None
                if n > 0:
                    z = step_noise[n - 1] if step_noise is not None else torch.randn_like(y)
                rc = L.b200tts_wavegrad_step(h, _lib.ptr(y), _lib.ptr(levels[n]), pe, pe_frames, ctypes.c_float(c1[n]),
                                             ctypes.c_float(c2[n]), ctypes.c_float(sigma[n - 1] if n > 0 else 0.0),
                                             _lib.ptr(z), b, t, _lib.ptr(ws), ctypes.c_size_t(ws.numel()), st)
                _lib.check(rc, "wavegrad_step")
        return y

    def compute_noise_level(self, beta):
        """wavegrad.py:160-176 (float64 numpy schedule cast to float32, then float32 torch on the CPU)."""
        self.num_steps = len(beta)
        alpha = 1 - beta
        alpha_hat = np.cumprod(alpha)
        noise_level = alpha_hat**0.5
        self.beta = torch.tensor(beta.astype(np.float32))
        self.alpha = torch.tensor(alpha.astype(np.float32))
        self.alpha_hat = torch.tensor(alpha_hat.astype(np.float32))
        self.noise_level = torch.tensor(noise_level.astype(np.float32))
        self.c1 = 1 / self.alpha**0.5
        self.c2 = (1 - self.alpha) / (1 - self.alpha_hat) ** 0.5
        self.sigma = ((1.0 - self.alpha_hat[:-1]) / (1.0 - self.alpha_hat[1:]) * self.beta[1:]) ** 0.5

    def load_noise_schedule(self, path):
        """wavegrad.py:122-124: ``beta`` from an ``.npy`` dict."""
        beta = np.load(path, allow_pickle=True).item()["beta"]
        self.compute_noise_level(beta)

    def apply_weight_norm(self):
        self._drop_handle()
        for blocks in (self.dblocks, self.film, self.ublocks):
            for layer in blocks:
                if len(layer.state_dict()) != 0:
                    layer.apply_weight_norm()
        self.x_conv = weight_norm(self.x_conv)
        self.out_conv = weight_norm(self.out_conv)
        self.y_conv = weight_norm(self.y_conv)

    def remove_weight_norm(self):
        self._drop_handle()
        for m in self.modules():
            if isinstance(m, nn.Conv1d) and is_parametrized(m, "weight"):
                remove_parametrizations(m, "weight")

    def load_checkpoint(self, config, checkpoint_path, eval=False, cache=False):  # pylint: disable=redefined-builtin
        """wavegrad.py:221-243: the state dict, then (eval) weight norm removed and the test schedule, else the train
        schedule."""
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        if eval:
            self.eval()
            assert not self.training
            if self.config.model_params.use_weight_norm:
                self.remove_weight_norm()
            s = config["test_noise_schedule"]
        else:
            s = config["train_noise_schedule"]
        self.compute_noise_level(np.linspace(s["min_val"], s["max_val"], s["num_steps"]))

    @staticmethod
    def init_from_config(config):
        return Wavegrad(config)
