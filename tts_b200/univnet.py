"""Drop-in for the UnivNet generator of the reference:

  UnivnetGenerator   <- TTS/vocoder/models/univnet_generator.py (LVCBlock, KernelPredictor: TTS/vocoder/layers/lvc_block.py)

Same constructor signature, same ``state_dict`` keys (the torch modules below are only parameter containers, weight-norm
parametrizations included, so reference checkpoints -- also ones with the legacy ``weight_g`` / ``weight_v`` keys -- load
unchanged), same ``forward`` (noise drawn with ``torch.randn`` on the CPU generator, then moved to the device, as the
reference does), ``inference`` (which, like the reference's, draws one noise tensor it discards before ``forward`` draws
its own, so a seed gives the reference's waveform), ``apply_weight_norm`` and ``remove_weight_norm``.  ``forward`` /
``inference`` also take ``noise=`` to supply the noise.

The arithmetic runs in libtts_b200.so (``b200tts_univnet_forward``): the kernel predictor on the conv engine, one
split-fp16 tensor-core GEMM per block for the predicted kernels, one fused split-fp16 tensor-core launch per LVC layer;
there is no PyTorch fallback.  The kernels take hidden_channels = 32 and lvc_kernel_size = 3 (the zoo model's),
kpnet_hidden_channels a multiple of 16 and an odd kpnet_conv_size; other values build the module (its state dict is the
reference's) but running it raises NotImplementedError naming the field.
"""
import ctypes

import torch
from torch import nn
from torch.nn.utils.parametrizations import weight_norm
from torch.nn.utils.parametrize import is_parametrized, remove_parametrizations

from . import _lib

RESIDUAL_CONVS = (1, 3, 6, 8, 11, 13)   # the Conv1d positions inside KernelPredictor.residual_conv


class _KernelPredictor(nn.Module):
    """Key layout of KernelPredictor (lvc_block.py)."""

    def __init__(self, cond_channels, conv_in_channels, conv_out_channels, conv_layers, conv_kernel_size,
                 kpnet_hidden_channels, kpnet_conv_size, kpnet_dropout):
        super().__init__()
        h, k = kpnet_hidden_channels, kpnet_conv_size
        padding = (k - 1) // 2
        self.input_conv = nn.Sequential(nn.Conv1d(cond_channels, h, 5, padding=2, bias=True), nn.LeakyReLU(0.1))
        layers = []
        for _ in range(3):
            layers += [nn.Dropout(kpnet_dropout)]
            for _ in range(2):
                layers += [nn.Conv1d(h, h, k, padding=padding, bias=True), nn.LeakyReLU(0.1)]
        self.residual_conv = nn.Sequential(*layers)
        l_w = conv_in_channels * conv_out_channels * conv_kernel_size * conv_layers
        self.kernel_conv = nn.Conv1d(h, l_w, k, padding=padding, bias=True)
        self.bias_conv = nn.Conv1d(h, conv_out_channels * conv_layers, k, padding=padding, bias=True)


class _LVCBlock(nn.Module):
    """Key layout of LVCBlock (lvc_block.py); ``convs`` is registered first, as there."""

    def __init__(self, in_channels, cond_channels, upsample_ratio, conv_layers, conv_kernel_size, cond_hop_length,
                 kpnet_hidden_channels, kpnet_conv_size, kpnet_dropout):
        super().__init__()
        self.cond_hop_length = cond_hop_length
        self.conv_layers = conv_layers
        self.convs = nn.ModuleList()
        u = upsample_ratio
        self.upsample = nn.ConvTranspose1d(in_channels, in_channels, kernel_size=2 * u, stride=u,
                                           padding=u // 2 + u % 2, output_padding=u % 2)
        self.kernel_predictor = _KernelPredictor(cond_channels, in_channels, 2 * in_channels, conv_layers,
                                                 conv_kernel_size, kpnet_hidden_channels, kpnet_conv_size, kpnet_dropout)
        for i in range(conv_layers):
            self.convs.append(nn.Conv1d(in_channels, in_channels, conv_kernel_size,
                                        padding=3 ** i * ((conv_kernel_size - 1) // 2), dilation=3 ** i))


class UnivnetGenerator(nn.Module):
    def __init__(self, in_channels, out_channels, hidden_channels, cond_channels, upsample_factors,
                 lvc_layers_each_block, lvc_kernel_size, kpnet_hidden_channels, kpnet_conv_size, dropout,
                 use_weight_norm=True):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.hidden_channels = hidden_channels
        self.cond_channels = cond_channels
        self.upsample_factors = list(upsample_factors)
        self.upsample_scale = 1
        for u in upsample_factors:
            self.upsample_scale *= int(u)
        self.lvc_block_nums = len(upsample_factors)
        self.lvc_layers_each_block = lvc_layers_each_block
        self.lvc_kernel_size = lvc_kernel_size
        self.kpnet_hidden_channels = kpnet_hidden_channels
        self.kpnet_conv_size = kpnet_conv_size
        self.dropout = dropout
        self.first_conv = nn.Conv1d(in_channels, hidden_channels, kernel_size=7, padding=3, dilation=1, bias=True)
        self.lvc_blocks = nn.ModuleList()
        hop = 1
        for u in upsample_factors:
            hop *= u
            self.lvc_blocks.append(_LVCBlock(hidden_channels, cond_channels, u, lvc_layers_each_block, lvc_kernel_size,
                                             hop, kpnet_hidden_channels, kpnet_conv_size, dropout))
        self.last_conv_layers = nn.ModuleList(
            [nn.Conv1d(hidden_channels, out_channels, kernel_size=7, padding=3, dilation=1, bias=True)])
        if use_weight_norm:
            self.apply_weight_norm()
        self._handle = None
        self._handle_device = None
        self._register_load_state_dict_pre_hook(lambda *a, **k: self._drop_handle())

    # ------------------------------------------------------------------ engine handle
    def _drop_handle(self):
        if getattr(self, "_handle", None) is not None:
            _lib.lib().b200tts_univnet_destroy(self._handle)
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

    def _check_supported(self):
        for name, ok, want in (("hidden_channels", self.hidden_channels == 32, "32"),
                               ("lvc_kernel_size", self.lvc_kernel_size == 3, "3"),
                               ("kpnet_hidden_channels", self.kpnet_hidden_channels % 16 == 0, "a multiple of 16"),
                               ("kpnet_conv_size", self.kpnet_conv_size % 2 == 1, "odd"),
                               ("upsample_factors", 1 <= len(self.upsample_factors) <= 8, "1 to 8 factors"),
                               ("lvc_layers_each_block", 1 <= self.lvc_layers_each_block <= 8, "1 to 8")):
            if not ok:
                raise NotImplementedError(f"tts_b200.UnivnetGenerator: {name} = {getattr(self, name)!r} (the kernels "
                                          f"take {name} {want})")
        if self.training and self.dropout > 0:
            raise NotImplementedError("tts_b200.UnivnetGenerator: dropout > 0 in training mode (inference only; call "
                                      ".eval())")

    def _ordered_weights(self):
        """Host fp32 tensors in the order include/tts_b200.h documents (weight norm folded by torch)."""
        def t(x):
            return x.detach().to(torch.float32).cpu().contiguous()

        out = [t(self.first_conv.weight), t(self.first_conv.bias)]
        for blk in self.lvc_blocks:
            kp = blk.kernel_predictor
            out += [t(blk.upsample.weight), t(blk.upsample.bias), t(kp.input_conv[0].weight), t(kp.input_conv[0].bias)]
            for i in RESIDUAL_CONVS:
                out += [t(kp.residual_conv[i].weight), t(kp.residual_conv[i].bias)]
            out += [t(kp.kernel_conv.weight), t(kp.kernel_conv.bias), t(kp.bias_conv.weight), t(kp.bias_conv.bias)]
            for conv in blk.convs:
                out += [t(conv.weight), t(conv.bias)]
        out += [t(self.last_conv_layers[0].weight), t(self.last_conv_layers[0].bias)]
        return out

    def _ensure_handle(self, device):
        if self._handle is not None and self._handle_device == device:
            return self._handle
        self._drop_handle()
        cfg = _lib.UnivnetConfigC()
        cfg.in_channels, cfg.out_channels = self.in_channels, self.out_channels
        cfg.hidden_channels, cfg.cond_channels = self.hidden_channels, self.cond_channels
        cfg.num_upsamples = len(self.upsample_factors)
        for i, u in enumerate(self.upsample_factors):
            cfg.upsample_factors[i] = int(u)
        cfg.lvc_layers, cfg.lvc_kernel_size = self.lvc_layers_each_block, self.lvc_kernel_size
        cfg.kpnet_hidden_channels, cfg.kpnet_conv_size = self.kpnet_hidden_channels, self.kpnet_conv_size
        tensors = self._ordered_weights()
        arr = (ctypes.c_void_p * len(tensors))(*[x.data_ptr() for x in tensors])
        handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            rc = _lib.lib().b200tts_univnet_create(ctypes.byref(cfg), arr, len(tensors), ctypes.byref(handle))
        _lib.check(rc, "univnet_create")
        self._handle, self._handle_device = handle, device
        return handle

    def _mel(self, c):
        self._check_supported()
        if c.dim() != 3 or c.shape[1] != self.cond_channels:
            raise RuntimeError(f"tts_b200.UnivnetGenerator: c must be [B, {self.cond_channels}, T], got {tuple(c.shape)}")
        _lib.require_cuda(c, "c")
        return c.to(torch.float32).contiguous()

    @torch.no_grad()
    def _run(self, c, noise):
        x = self._mel(c)
        b, _, t = x.shape
        if noise is None:   # the reference's draw: CPU generator, then a copy to the device
            noise = torch.randn([b, self.in_channels, t])
        if tuple(noise.shape) != (b, self.in_channels, t):
            raise ValueError(f"tts_b200.UnivnetGenerator: noise must be {(b, self.in_channels, t)}, got "
                             f"{tuple(noise.shape)}")
        noise = noise.to(device=x.device, dtype=torch.float32).contiguous()
        h = self._ensure_handle(x.device)
        L = _lib.lib()
        with torch.cuda.device(x.device):
            out = torch.empty((b, self.out_channels, t * self.upsample_scale), dtype=torch.float32, device=x.device)
            ws = _lib.workspace(x.device, L.b200tts_univnet_workspace_bytes(h, b, t), "univnet")
            rc = L.b200tts_univnet_forward(h, _lib.ptr(x), _lib.ptr(noise), b, t, _lib.ptr(out), _lib.ptr(ws),
                                           ctypes.c_size_t(ws.numel()), _lib.stream_ptr(x.device))
        _lib.check(rc, "univnet_forward")
        return out

    # ------------------------------------------------------------------ test aids
    @torch.no_grad()
    def predict(self, block, c):
        """Block ``block``'s kernel predictor as the layers read it: c [B, cond, T] (CUDA) -> (kernels
        [B, T, L, 64 (co), 3 (tap), 32 (ci)], biases [B, T, L, 64]) -- frame-major, the layout of b200tts_univnet_predict."""
        x = self._mel(c)
        b, _, t = x.shape
        h = self._ensure_handle(x.device)
        L = _lib.lib()
        n = self.lvc_layers_each_block
        with torch.cuda.device(x.device):
            pred = torch.empty((b, t, n * (64 * 96 + 64)), dtype=torch.float32, device=x.device)
            ws = _lib.workspace(x.device, L.b200tts_univnet_workspace_bytes(h, b, t), "univnet")
            rc = L.b200tts_univnet_predict(h, block, _lib.ptr(x), b, t, _lib.ptr(pred), _lib.ptr(ws),
                                           ctypes.c_size_t(ws.numel()), _lib.stream_ptr(x.device))
        _lib.check(rc, "univnet_predict")
        return pred[..., : n * 6144].view(b, t, n, 64, 3, 32), pred[..., n * 6144:].view(b, t, n, 64)

    # ------------------------------------------------------------------ reference API
    def forward(self, c, noise=None):
        """c [B, cond_channels, T] (CUDA) -> waveform [B, out_channels, T * prod(upsample_factors)]
        (univnet_generator.py forward).  ``noise`` [B, in_channels, T] replaces the ``torch.randn`` draw."""
        return self._run(c, noise)

    @torch.no_grad()
    def inference(self, c, noise=None):
        """The reference's inference: one ``torch.randn([B, in_channels, T])`` draw that is discarded, then ``forward``
        (which draws again); with ``noise`` given, neither draw happens and ``noise`` is used."""
        c = c.to(self.first_conv.bias.device)
        if noise is None:
            self._mel(c)    # the checks come before the draws, as a failing call should not move the generator
            torch.randn([c.shape[0], self.in_channels, c.shape[2]])
        return self._run(c, noise)

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
        """A bare-generator checkpoint ({"model": state_dict}); ``eval`` also removes weight norm."""
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        if eval:
            self.eval()
            self.remove_weight_norm()
