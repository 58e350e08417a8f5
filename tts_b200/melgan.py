"""Drop-ins for the MelGAN generator family of the reference:

  MelganGenerator            <- TTS/vocoder/models/melgan_generator.py:9-96 (ResidualStack: TTS/vocoder/layers/melgan.py)
  MultibandMelganGenerator   <- TTS/vocoder/models/multiband_melgan_generator.py:7-43
  FullbandMelganGenerator    <- TTS/vocoder/models/fullband_melgan_generator.py:6-33
  PQMF                       <- TTS/vocoder/layers/pqmf.py:9-53 (synthesis only; analysis is training-side)

Same constructor signatures and defaults, same ``state_dict`` keys (the torch modules below are only parameter containers,
weight-norm parametrizations and the PQMF buffers included, so reference checkpoints load unchanged), same ``forward``
(the generator layers: the 4 band signals of a multi-band generator), ``inference`` (replicate pad of
``inference_padding = 2`` frames, the layers and, for the multi-band generator, PQMF synthesis; the padded output is not
trimmed), ``pqmf_synthesis``, ``remove_weight_norm`` and ``load_checkpoint``.  The arithmetic runs in libtts_b200.so
(``b200tts_melgan_forward`` / ``b200tts_pqmf_synthesis``); there is no PyTorch fallback.
"""
import ctypes

import numpy as np
import torch
from scipy import signal
from torch import nn
from torch.nn.utils.parametrizations import weight_norm
from torch.nn.utils.parametrize import is_parametrized, remove_parametrizations

from . import _lib

ACT_SLOPE = 0.2


class _ResidualStack(nn.Module):
    """Parameter container with the key layout of ResidualStack (layers/melgan.py:6-31): ``blocks.M`` =
    (LeakyReLU, ReflectionPad1d, dilated conv, LeakyReLU, 1x1 conv), ``shortcuts.M`` = 1x1 conv."""

    def __init__(self, channels, num_res_blocks, kernel_size):
        super().__init__()
        assert (kernel_size - 1) % 2 == 0, " [!] kernel_size has to be odd."
        self.blocks = nn.ModuleList()
        for m in range(num_res_blocks):
            dilation = kernel_size ** m
            self.blocks.append(nn.Sequential(
                nn.LeakyReLU(ACT_SLOPE),
                nn.ReflectionPad1d((kernel_size - 1) // 2 * dilation),
                weight_norm(nn.Conv1d(channels, channels, kernel_size=kernel_size, dilation=dilation, bias=True)),
                nn.LeakyReLU(ACT_SLOPE),
                weight_norm(nn.Conv1d(channels, channels, kernel_size=1, bias=True))))
        self.shortcuts = nn.ModuleList(
            [weight_norm(nn.Conv1d(channels, channels, kernel_size=1, bias=True)) for _ in range(num_res_blocks)])

    def convs(self):
        """Per block: dilated conv, 1x1 conv, shortcut (the order include/tts_b200.h documents)."""
        out = []
        for block, shortcut in zip(self.blocks, self.shortcuts):
            out += [block[2], block[4], shortcut]
        return out


class PQMF(nn.Module):
    """Pseudo-QMF filter bank (pqmf.py:9-53): the ``H`` / ``G`` / ``updown_filter`` buffers are built from a Kaiser-window
    ``scipy.signal.firwin`` prototype exactly as the reference builds them; ``synthesis`` runs the polyphase kernel."""

    def __init__(self, N=4, taps=62, cutoff=0.15, beta=9.0):
        super().__init__()
        self.N, self.taps, self.cutoff, self.beta = N, taps, cutoff, beta
        proto = signal.firwin(taps + 1, cutoff, window=("kaiser", beta))
        H = np.zeros((N, len(proto)))
        G = np.zeros((N, len(proto)))
        offset = np.arange(taps + 1) - ((taps - 1) / 2)    # centred on (taps - 1) / 2, as in the reference
        for k in range(N):
            arg = (2 * k + 1) * (np.pi / (2 * N)) * offset
            phase = (-1) ** k * np.pi / 4
            H[k] = 2 * proto * np.cos(arg + phase)
            G[k] = 2 * proto * np.cos(arg - phase)
        self.register_buffer("H", torch.from_numpy(H[:, None, :]).float())
        self.register_buffer("G", torch.from_numpy(G[None, :, :]).float())
        updown = torch.zeros((N, N, N)).float()
        for k in range(N):
            updown[k, k, 0] = 1.0
        self.register_buffer("updown_filter", updown)
        self.pad_fn = nn.ConstantPad1d(taps // 2, 0.0)

    def forward(self, x):
        return self.analysis(x)

    def analysis(self, x):
        raise NotImplementedError("tts_b200.PQMF.analysis: PQMF analysis is only used in training")

    @torch.no_grad()
    def synthesis(self, x, peak=None):
        """x [B, N, Tb] (CUDA) -> [B, 1, N * Tb - taps % 2] (pqmf.py:50-53; an odd tap count loses a sample, as there).
        ``peak``: optional zeroed int32[1] device word that max|y| is folded into (``tts_b200.vocoder.wav_to_int16``)."""
        _lib.require_cuda(x, "x")
        x = x.to(torch.float32).contiguous()
        b, n, tb = x.shape
        if n != self.N:
            raise ValueError(f"tts_b200.PQMF.synthesis: expected {self.N} bands, got {n}")
        g = self.G.to(device=x.device, dtype=torch.float32).contiguous()
        y = torch.empty((b, 1, n * tb - self.taps % 2), dtype=torch.float32, device=x.device)   # as conv1d(padding=taps//2)
        with torch.cuda.device(x.device):
            rc = _lib.lib().b200tts_pqmf_synthesis(_lib.ptr(x), b, n, tb, _lib.ptr(g), self.taps, _lib.ptr(y),
                                                   _lib.ptr(peak), _lib.stream_ptr(x.device))
        _lib.check(rc, "pqmf_synthesis")
        return y


class MelganGenerator(nn.Module):
    def __init__(self, in_channels=80, out_channels=1, proj_kernel=7, base_channels=512, upsample_factors=(8, 8, 2, 2),
                 res_kernel=3, num_res_blocks=3):
        super().__init__()
        assert (proj_kernel - 1) % 2 == 0, " [!] proj_kernel should be an odd number."
        base_padding = (proj_kernel - 1) // 2
        self.inference_padding = 2
        self._cfg = dict(in_channels=in_channels, out_channels=out_channels, proj_kernel=proj_kernel,
                         base_channels=base_channels, upsample_factors=list(upsample_factors), res_kernel=res_kernel,
                         num_res_blocks=num_res_blocks)
        layers = [nn.ReflectionPad1d(base_padding),
                  weight_norm(nn.Conv1d(in_channels, base_channels, kernel_size=proj_kernel, stride=1, bias=True))]
        ch = base_channels
        for u in upsample_factors:
            out_ch = ch // 2
            layers += [nn.LeakyReLU(ACT_SLOPE),
                       weight_norm(nn.ConvTranspose1d(ch, out_ch, u * 2, stride=u, padding=u // 2 + u % 2,
                                                      output_padding=u % 2, bias=True)),
                       _ResidualStack(out_ch, num_res_blocks, res_kernel)]
            ch = out_ch
        layers += [nn.LeakyReLU(ACT_SLOPE), nn.ReflectionPad1d(base_padding),
                   weight_norm(nn.Conv1d(ch, out_channels, proj_kernel, stride=1, bias=True)), nn.Tanh()]
        self.layers = nn.Sequential(*layers)
        self._handle = None
        self._handle_device = None
        # a parent's load_state_dict recurses through _load_from_state_dict, never a child's override: drop the packed
        # handle from a pre-hook (as HifiganGenerator does)
        self._register_load_state_dict_pre_hook(lambda *a, **k: self._drop_handle())

    # ------------------------------------------------------------------ engine handle
    def _pqmf(self):
        return None

    def _drop_handle(self):
        if getattr(self, "_handle", None) is not None:
            _lib.lib().b200tts_melgan_destroy(self._handle)
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

    def _ordered_weights(self):
        """Host fp32 tensors in the order include/tts_b200.h documents (weight norm folded by torch)."""
        def wb(m):
            return [m.weight.detach().to(torch.float32).cpu().contiguous(),
                    m.bias.detach().to(torch.float32).cpu().contiguous()]

        n_up = len(self._cfg["upsample_factors"])
        out = wb(self.layers[1])
        for s in range(n_up):
            out += wb(self.layers[3 + 3 * s])
            for conv in self.layers[4 + 3 * s].convs():
                out += wb(conv)
        out += wb(self.layers[3 * n_up + 4])
        pq = self._pqmf()
        if pq is not None:
            out.append(pq.G.detach().to(torch.float32).cpu().contiguous())
        return out

    def _ensure_handle(self, device):
        if self._handle is not None and self._handle_device == device:
            return self._handle
        self._drop_handle()
        c = self._cfg
        cfg = _lib.MelganConfigC()
        cfg.in_channels, cfg.out_channels, cfg.base_channels = c["in_channels"], c["out_channels"], c["base_channels"]
        cfg.proj_kernel, cfg.res_kernel, cfg.num_res_blocks = c["proj_kernel"], c["res_kernel"], c["num_res_blocks"]
        if not 1 <= len(c["upsample_factors"]) <= 8:
            raise ValueError("tts_b200: 1 to 8 upsample factors are supported")
        cfg.num_upsamples = len(c["upsample_factors"])
        for i, u in enumerate(c["upsample_factors"]):
            cfg.upsample_factors[i] = u
        pq = self._pqmf()
        cfg.pqmf_bands, cfg.pqmf_taps = (pq.N, pq.taps) if pq is not None else (0, 0)
        tensors = self._ordered_weights()
        arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            rc = _lib.lib().b200tts_melgan_create(ctypes.byref(cfg), arr, len(tensors), ctypes.byref(handle))
        _lib.check(rc, "melgan_create")
        self._handle, self._handle_device = handle, device
        return handle

    @torch.no_grad()
    def _run(self, c, synthesize, peak=None):
        _lib.require_cuda(c, "c")
        x = c.to(torch.float32).contiguous()
        b, cin, t = x.shape
        if cin != self._cfg["in_channels"]:
            raise ValueError(f"expected {self._cfg['in_channels']} input channels, got {cin}")
        h = self._ensure_handle(x.device)
        L = _lib.lib()
        with torch.cuda.device(x.device):
            tout = L.b200tts_melgan_out_len(h, t)
            pq = self._pqmf()
            shape = (b, 1, pq.N * tout - pq.taps % 2) if synthesize else (b, self._cfg["out_channels"], tout)
            out = torch.empty(shape, dtype=torch.float32, device=x.device)
            nbytes = L.b200tts_melgan_workspace_bytes(h, b, t)
            ws = _lib.workspace(x.device, nbytes, "melgan")
            rc = L.b200tts_melgan_forward(h, _lib.ptr(x), b, t, int(synthesize), _lib.ptr(out), _lib.ptr(peak),
                                          _lib.ptr(ws), ctypes.c_size_t(ws.numel()), _lib.stream_ptr(x.device))
        _lib.check(rc, "melgan_forward")   # RuntimeError (torch's type) for an input too short for a reflect pad
        return out

    # ------------------------------------------------------------------ reference API
    def forward(self, c, peak=None):
        """c [B, in_channels, T] (CUDA) -> ``self.layers(c)``: [B, out_channels, T * prod(upsample_factors)]
        (melgan_generator.py:72-73).  ``peak``: optional zeroed int32[1] device word conv_post folds max|y| into."""
        return self._run(c, False, peak)

    def _padded(self, c):
        from .vocoder import AudioNorm, vocoder_input
        c = c.to(self.layers[1].bias.device)
        # the replicate pad comes from the hand-off kernel, as in HifiganGenerator.inference
        return vocoder_input(c, AudioNorm.identity(), AudioNorm.identity(), padding=self.inference_padding)

    @torch.no_grad()
    def inference(self, c, peak=None):
        """Replicate-pad ``inference_padding`` (2) frames each side, then the layers (melgan_generator.py:75-78)."""
        return self._run(self._padded(c), False, peak)

    def remove_weight_norm(self):
        self._drop_handle()
        for m in self.modules():
            if isinstance(m, (nn.Conv1d, nn.ConvTranspose1d)) and is_parametrized(m, "weight"):
                remove_parametrizations(m, "weight")

    def load_checkpoint(self, config, checkpoint_path, eval=False, cache=False):  # pylint: disable=redefined-builtin
        """melgan_generator.py:88-96."""
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        if eval:
            self.eval()
            assert not self.training
            self.remove_weight_norm()


class MultibandMelganGenerator(MelganGenerator):
    """multiband_melgan_generator.py:7-43: ``forward`` returns the 4 band signals, ``inference`` the PQMF-synthesised
    waveform [B, 1, 4 * T * prod(upsample_factors)] (one engine call: the layers, then the synthesis kernel)."""

    def __init__(self, in_channels=80, out_channels=4, proj_kernel=7, base_channels=384, upsample_factors=(2, 8, 2, 2),
                 res_kernel=3, num_res_blocks=3):
        super().__init__(in_channels=in_channels, out_channels=out_channels, proj_kernel=proj_kernel,
                         base_channels=base_channels, upsample_factors=upsample_factors, res_kernel=res_kernel,
                         num_res_blocks=num_res_blocks)
        self.pqmf_layer = PQMF(N=4, taps=62, cutoff=0.15, beta=9.0)

    def _pqmf(self):
        return self.pqmf_layer

    def pqmf_analysis(self, x):
        return self.pqmf_layer.analysis(x)

    def pqmf_synthesis(self, x, peak=None):
        return self.pqmf_layer.synthesis(x, peak)

    @torch.no_grad()
    def inference(self, cond_features, peak=None):
        return self._run(self._padded(cond_features), True, peak)


class FullbandMelganGenerator(MelganGenerator):
    """fullband_melgan_generator.py:6-33."""

    def __init__(self, in_channels=80, out_channels=1, proj_kernel=7, base_channels=512, upsample_factors=(2, 8, 2, 2),
                 res_kernel=3, num_res_blocks=4):
        super().__init__(in_channels=in_channels, out_channels=out_channels, proj_kernel=proj_kernel,
                         base_channels=base_channels, upsample_factors=upsample_factors, res_kernel=res_kernel,
                         num_res_blocks=num_res_blocks)
