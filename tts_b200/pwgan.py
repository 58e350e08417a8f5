"""Drop-in for the Parallel WaveGAN generator of the reference:

  ParallelWaveganGenerator   <- TTS/vocoder/models/parallel_wavegan_generator.py:12-178 (ResidualBlock:
                                TTS/vocoder/layers/parallel_wavegan.py, ConvUpsample: TTS/vocoder/layers/upsample.py)

Same constructor signature and defaults, same ``state_dict`` keys (the torch modules below are only parameter containers,
weight-norm parametrizations included, so reference checkpoints -- also ones with the legacy ``weight_g`` / ``weight_v``
keys -- load unchanged), same ``forward`` (noise drawn with ``torch.randn`` on the CPU generator, then moved to the
device, as the reference does), ``inference`` (replicate pad of ``inference_padding`` frames), ``apply_weight_norm``,
``remove_weight_norm`` and ``load_checkpoint``.  ``forward`` / ``inference`` also take ``noise=`` to supply the noise.

The arithmetic runs in libtts_b200.so (``b200tts_pwgan_forward``): one fused split-fp16 tensor-core launch per residual
layer, with the upsampled conditioning folded into it; there is no PyTorch fallback.  The kernel takes the shapes
``setup_generator`` builds (64 residual / 128 gate / 64 skip channels, kernel 3, one noise channel in and one waveform
channel out, convs with bias); other shapes raise NotImplementedError naming the field.
"""
import ctypes

import torch
from torch import nn
from torch.nn.utils.parametrizations import weight_norm
from torch.nn.utils.parametrize import is_parametrized, remove_parametrizations

from . import _lib

MEL_CHANNELS = 80   # ConvUpsample is built with its default aux_channels, whatever the generator's aux_channels


class _Stretch2d(nn.Module):
    """Stretch2d (upsample.py:5-19): nearest interpolation, no parameters."""

    def __init__(self, x_scale, y_scale, mode="nearest"):
        super().__init__()
        self.x_scale, self.y_scale, self.mode = x_scale, y_scale, mode


class _UpsampleNetwork(nn.Module):
    """Key layout of UpsampleNetwork (upsample.py:22-71): ``up_layers`` = (Stretch2d, Conv2d(1, 1, (1, 2u + 1))) per
    factor, no nonlinearity."""

    def __init__(self, upsample_factors):
        super().__init__()
        self.up_layers = nn.ModuleList()
        for scale in upsample_factors:
            self.up_layers += [_Stretch2d(scale, 1),
                               nn.Conv2d(1, 1, kernel_size=(1, scale * 2 + 1), padding=(0, scale), bias=False)]


class _ConvUpsample(nn.Module):
    """Key layout of ConvUpsample (upsample.py:74-111) at aux_context_window = 0: ``conv_in`` is an 80 -> 80 1x1 conv."""

    def __init__(self, upsample_factors, aux_channels=MEL_CHANNELS):
        super().__init__()
        self.conv_in = nn.Conv1d(aux_channels, aux_channels, kernel_size=1, bias=False)
        self.upsample = _UpsampleNetwork(upsample_factors)


class _ResidualBlock(nn.Module):
    """Key layout of ResidualBlock (parallel_wavegan.py:5-47)."""

    def __init__(self, kernel_size, res_channels, gate_channels, skip_channels, aux_channels, dilation, bias):
        super().__init__()
        padding = (kernel_size - 1) // 2 * dilation
        self.conv = nn.Conv1d(res_channels, gate_channels, kernel_size, padding=padding, dilation=dilation, bias=bias)
        self.conv1x1_aux = nn.Conv1d(aux_channels, gate_channels, 1, bias=False) if aux_channels > 0 else None
        self.conv1x1_out = nn.Conv1d(gate_channels // 2, res_channels, 1, bias=bias)
        self.conv1x1_skip = nn.Conv1d(gate_channels // 2, skip_channels, 1, bias=bias)


class ParallelWaveganGenerator(nn.Module):
    # pylint: disable=dangerous-default-value
    def __init__(self, in_channels=1, out_channels=1, kernel_size=3, num_res_blocks=30, stacks=3, res_channels=64,
                 gate_channels=128, skip_channels=64, aux_channels=80, dropout=0.0, bias=True, use_weight_norm=True,
                 upsample_factors=[4, 4, 4, 4], inference_padding=2):
        super().__init__()
        for name, value, want in (("in_channels", in_channels, 1), ("out_channels", out_channels, 1),
                                  ("kernel_size", kernel_size, 3), ("res_channels", res_channels, 64),
                                  ("gate_channels", gate_channels, 128), ("skip_channels", skip_channels, 64),
                                  ("bias", bias, True)):
            if value != want:
                raise NotImplementedError(f"tts_b200.ParallelWaveganGenerator: {name} = {value!r} (the kernel takes "
                                          f"{name} = {want!r}, as setup_generator builds it)")
        assert num_res_blocks % stacks == 0
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.aux_channels = aux_channels
        self.num_res_blocks = num_res_blocks
        self.stacks = stacks
        self.kernel_size = kernel_size
        self.upsample_factors = upsample_factors
        self.upsample_scale = 1
        for u in upsample_factors:
            self.upsample_scale *= int(u)
        self.inference_padding = inference_padding
        self.use_weight_norm = use_weight_norm
        layers_per_stack = num_res_blocks // stacks
        self.first_conv = nn.Conv1d(in_channels, res_channels, kernel_size=1, bias=True)
        self.upsample_net = _ConvUpsample(upsample_factors)
        self.conv_layers = nn.ModuleList(
            [_ResidualBlock(kernel_size, res_channels, gate_channels, skip_channels, aux_channels,
                            2 ** (layer % layers_per_stack), bias) for layer in range(num_res_blocks)])
        self.last_conv_layers = nn.ModuleList([nn.ReLU(inplace=True),
                                               nn.Conv1d(skip_channels, skip_channels, kernel_size=1, bias=True),
                                               nn.ReLU(inplace=True),
                                               nn.Conv1d(skip_channels, out_channels, kernel_size=1, bias=True)])
        if use_weight_norm:
            self.apply_weight_norm()
        self._handle = None
        self._handle_device = None
        self._register_load_state_dict_pre_hook(lambda *a, **k: self._drop_handle())

    # ------------------------------------------------------------------ engine handle
    def _drop_handle(self):
        if getattr(self, "_handle", None) is not None:
            _lib.lib().b200tts_pwgan_destroy(self._handle)
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
        def t(x):
            return x.detach().to(torch.float32).cpu().contiguous()

        out = [t(self.first_conv.weight), t(self.first_conv.bias), t(self.upsample_net.conv_in.weight)]
        out += [t(m.weight) for m in self.upsample_net.upsample.up_layers if isinstance(m, nn.Conv2d)]
        for blk in self.conv_layers:
            out += [t(blk.conv.weight), t(blk.conv.bias), t(blk.conv1x1_aux.weight), t(blk.conv1x1_out.weight),
                    t(blk.conv1x1_out.bias), t(blk.conv1x1_skip.weight), t(blk.conv1x1_skip.bias)]
        for i in (1, 3):
            out += [t(self.last_conv_layers[i].weight), t(self.last_conv_layers[i].bias)]
        return out

    def _ensure_handle(self, device):
        if self._handle is not None and self._handle_device == device:
            return self._handle
        self._drop_handle()
        if not 1 <= len(self.upsample_factors) <= 8:
            raise ValueError("tts_b200: 1 to 8 upsample factors are supported")
        cfg = _lib.PwganConfigC()
        cfg.num_res_blocks, cfg.stacks, cfg.num_upsamples = self.num_res_blocks, self.stacks, len(self.upsample_factors)
        for i, u in enumerate(self.upsample_factors):
            cfg.upsample_factors[i] = int(u)
        tensors = self._ordered_weights()
        arr = (ctypes.c_void_p * len(tensors))(*[x.data_ptr() for x in tensors])
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            rc = _lib.lib().b200tts_pwgan_create(ctypes.byref(cfg), arr, len(tensors), ctypes.byref(handle))
        _lib.check(rc, "pwgan_create")
        self._handle, self._handle_device = handle, device
        return handle

    @torch.no_grad()
    def _run(self, c, pad, noise):
        if self.conv_layers[0].conv1x1_aux is None or self.aux_channels != MEL_CHANNELS or c.dim() != 3 \
                or c.shape[1] != MEL_CHANNELS:
            # the reference's upsampler always has 80 channels: any other count fails in its convs (RuntimeError)
            raise RuntimeError(f"tts_b200.ParallelWaveganGenerator: the conditioning upsampler takes {MEL_CHANNELS} "
                               f"channels (aux_channels = {self.aux_channels}, input {tuple(c.shape)})")
        _lib.require_cuda(c, "c")
        x = c.to(torch.float32).contiguous()
        b, _, t = x.shape
        samples = (t + 2 * pad) * self.upsample_scale
        if noise is None:   # the reference's draw: CPU generator, then a copy to the device
            noise = torch.randn([b, 1, samples])
        if tuple(noise.shape) != (b, 1, samples):
            raise ValueError(f"tts_b200.ParallelWaveganGenerator: noise must be {(b, 1, samples)}, got {tuple(noise.shape)}")
        noise = noise.to(device=x.device, dtype=torch.float32).contiguous()
        h = self._ensure_handle(x.device)
        L = _lib.lib()
        with torch.cuda.device(x.device):
            out = torch.empty((b, 1, samples), dtype=torch.float32, device=x.device)
            ws = _lib.workspace(x.device, L.b200tts_pwgan_workspace_bytes(h, b, t + 2 * pad), "pwgan")
            rc = L.b200tts_pwgan_forward(h, _lib.ptr(x), _lib.ptr(noise), b, t, pad, _lib.ptr(out), _lib.ptr(ws),
                                         ctypes.c_size_t(ws.numel()), _lib.stream_ptr(x.device))
        _lib.check(rc, "pwgan_forward")
        return out

    def min_frames(self, device):
        """The shortest conditioning input (frames, after any pad) the upsampler tables take."""
        return int(_lib.lib().b200tts_pwgan_min_frames(self._ensure_handle(device)))

    @torch.no_grad()
    def upsample(self, a):
        """The conditioning upsampler's linear map as the layers apply it, on a CUDA [rows, Tf] tensor ->
        [rows, Tf * prod(upsample_factors)] (the stages of ConvUpsample.upsample without conv_in)."""
        _lib.require_cuda(a, "a")
        a = a.to(torch.float32).contiguous()
        rows, tf = a.shape
        h = self._ensure_handle(a.device)
        out = torch.empty((rows, tf * self.upsample_scale), dtype=torch.float32, device=a.device)
        with torch.cuda.device(a.device):
            rc = _lib.lib().b200tts_pwgan_upsample(h, _lib.ptr(a), rows, tf, _lib.ptr(out), _lib.stream_ptr(a.device))
        _lib.check(rc, "pwgan_upsample")
        return out

    # ------------------------------------------------------------------ reference API
    def forward(self, c, noise=None):
        """c [B, 80, T] (CUDA) -> waveform [B, 1, T * prod(upsample_factors)] (parallel_wavegan_generator.py:93-121).
        ``noise`` [B, 1, T * prod(upsample_factors)] replaces the ``torch.randn`` draw.

        Unlike the reference, T must be at least ``min_frames(device)`` (at most 5 for the default factors and for
        [3, 5, 4]): the upsampler tables are exact only down to that length.  ``inference`` pads ``inference_padding``
        frames each side first, so there T >= 1 works for those factors.  A shorter input raises RuntimeError before
        anything is launched."""
        return self._run(c, 0, noise)

    @torch.no_grad()
    def inference(self, c, noise=None):
        """Replicate-pad ``inference_padding`` frames each side, then ``forward`` (:123-127); ``noise`` is
        [B, 1, (T + 2 inference_padding) * prod(upsample_factors)]."""
        c = c.to(self.first_conv.weight.device)
        return self._run(c, self.inference_padding, noise)

    def remove_weight_norm(self):
        self._drop_handle()
        for m in self.modules():
            if isinstance(m, (nn.Conv1d, nn.Conv2d)) and is_parametrized(m, "weight"):
                remove_parametrizations(m, "weight")

    def apply_weight_norm(self):
        self._drop_handle()
        for m in self.modules():
            if isinstance(m, (nn.Conv1d, nn.Conv2d)):
                weight_norm(m)

    def load_checkpoint(self, config, checkpoint_path, eval=False, cache=False):  # pylint: disable=redefined-builtin
        """parallel_wavegan_generator.py:158-168."""
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        if eval:
            self.eval()
            assert not self.training
            if self.use_weight_norm:
                self.remove_weight_norm()
