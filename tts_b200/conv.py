"""One conv layer of the path with its fused prologue / epilogue (``b200tts_conv1d_*``): the building block the
HiFiGAN / flow / posterior engines run on, exposed so a layer can be checked or reused on its own.

Replaces one ``F.conv1d`` / ``F.conv_transpose1d`` call plus the element-wise ops around it, e.g. the ResBlock1 step
``xt = F.leaky_relu(x, 0.1); xt = c(xt); x = xt + x`` (/root/reference/TTS/vocoder/models/hifigan_generator.py:93-99):

    y = ((conv(leaky_relu(x, in_slope)) + bias) + residual) * scale [+ y if accumulate] / post_div
"""
import ctypes

import torch

from . import _lib


class FusedConv1d:
    """weight [Cout,Cin,K] (or [Cin,Cout,K] with ``transposed=True``), bias [Cout] or None -- host or device tensors;
    the packed device copy is created on first use per device.  ``precision`` "bf16" / "fp16" runs the tensor-core
    kernels with 16-bit operands (fp32 accumulation; layers with Cin % 16 != 0 stay 3xTF32); "f16x3" with the split-fp16
    product the HiFiGAN decoder uses by default (fp32-class accuracy for activations below 65504 in magnitude, same
    Cin rule); "fp32" (3xTF32 on the tensor cores) and "tf32x3" are the ``tensor_cores`` setting as given.  ``padding_mode`` mirrors ``nn.Conv1d``'s: "zeros" (default) or "reflect"
    (``nn.ReflectionPad1d(padding)`` then an unpadded conv, read straight from x by the kernels: no padded copy; needs
    ``padding = dilation * (K - 1) / 2``, ``padding <= T - 1`` and a non-transposed conv)."""

    def __init__(self, weight, bias=None, dilation=1, padding=0, transposed=False, stride=1, tensor_cores=True,
                 precision="fp32", padding_mode="zeros"):
        self.weight = weight.detach().to(torch.float32).cpu().contiguous()
        self.bias = None if bias is None else bias.detach().to(torch.float32).cpu().contiguous()
        self.dilation, self.padding, self.transposed, self.stride = int(dilation), int(padding), bool(transposed), int(stride)
        self.tensor_cores = bool(tensor_cores)
        self.precision = precision
        if padding_mode not in _lib.PADDING_MODES:
            raise ValueError(f"tts_b200.FusedConv1d: padding_mode must be one of {sorted(_lib.PADDING_MODES)}, "
                             f"got {padding_mode!r}")
        self.padding_mode = padding_mode
        if _lib.precision_id(precision) != 0 and not self.tensor_cores:
            raise ValueError("tts_b200.FusedConv1d: a precision other than fp32 needs tensor_cores=True")
        if transposed:
            self.cin, self.cout, self.k = self.weight.shape
        else:
            self.cout, self.cin, self.k = self.weight.shape
        self._handles = {}

    def __del__(self):
        try:
            for h in self._handles.values():
                _lib.lib().b200tts_conv1d_destroy(h)
        except Exception:  # pragma: no cover - interpreter shutdown
            pass

    def _handle(self, device):
        h = self._handles.get(device)
        if h is None:
            cfg = _lib.Conv1dConfigC(self.cin, self.cout, self.k, self.dilation, self.padding, int(self.transposed), self.stride)
            out = ctypes.c_void_p()
            with torch.cuda.device(device):
                if self.padding_mode != "zeros":
                    rc = _lib.lib().b200tts_conv1d_create_padded(
                        ctypes.byref(cfg), _lib.ptr(self.weight), _lib.ptr(self.bias), int(self.tensor_cores),
                        _lib.precision_id(self.precision), _lib.PADDING_MODES[self.padding_mode], ctypes.byref(out))
                elif self.precision == "fp32":
                    rc = _lib.lib().b200tts_conv1d_create(ctypes.byref(cfg), _lib.ptr(self.weight), _lib.ptr(self.bias),
                                                          int(self.tensor_cores), ctypes.byref(out))
                else:
                    rc = _lib.lib().b200tts_conv1d_create_ex(ctypes.byref(cfg), _lib.ptr(self.weight), _lib.ptr(self.bias),
                                                             _lib.precision_id(self.precision), ctypes.byref(out))
            _lib.check(rc, "conv1d_create")
            self._handles[device] = h = out
        return h

    @torch.no_grad()
    def __call__(self, x, in_slope=1.0, residual=None, scale=1.0, accumulate_into=None, post_div=1.0, tanh=False,
                 peak=None):
        """``tanh=True``: y = tanh(conv(leaky_relu(x)) + bias) (no residual / accumulate), and ``peak`` (optional zeroed
        int32[1] device word) folds max|y| in.  With reflection padding, ``tanh`` or ``peak``, a float32 x whose time
        axis is contiguous is read in place through its batch / channel strides."""
        _lib.require_cuda(x, "x")
        strided = self.padding_mode != "zeros" or tanh or peak is not None
        if tanh and (residual is not None or accumulate_into is not None):
            raise ValueError("tts_b200.FusedConv1d: the tanh epilogue takes no residual / accumulate")
        if peak is not None and not tanh:
            raise ValueError("tts_b200.FusedConv1d: peak needs tanh=True")
        x = x.to(torch.float32)
        if not strided or x.dim() != 3 or x.stride(-1) != 1:
            x = x.contiguous()
        b, cin, t = x.shape
        if cin != self.cin:
            raise ValueError(f"tts_b200.FusedConv1d: expected {self.cin} input channels, got {cin}")
        h = self._handle(x.device)
        L = _lib.lib()
        tout = L.b200tts_conv1d_out_len(h, t)
        if accumulate_into is not None:
            y = accumulate_into
            if tuple(y.shape) != (b, self.cout, tout) or not y.is_contiguous():
                raise ValueError("tts_b200.FusedConv1d: accumulate_into has the wrong shape")
        else:
            y = torch.empty((b, self.cout, tout), dtype=torch.float32, device=x.device)
        if residual is not None:
            residual = residual.to(torch.float32).contiguous()
            if tuple(residual.shape) != (b, self.cout, tout):
                raise ValueError("tts_b200.FusedConv1d: residual has the wrong shape")
        with torch.cuda.device(x.device):
            if strided:
                rc = L.b200tts_conv1d_forward_strided(h, _lib.ptr(x), ctypes.c_longlong(x.stride(0)), x.stride(1), b, t,
                                                      ctypes.c_float(in_slope), _lib.ptr(residual), ctypes.c_float(scale),
                                                      0 if accumulate_into is None else 1, ctypes.c_float(post_div),
                                                      int(bool(tanh)), _lib.ptr(y), _lib.ptr(peak),
                                                      _lib.stream_ptr(x.device))
            else:
                rc = L.b200tts_conv1d_forward(h, _lib.ptr(x), b, t, ctypes.c_float(in_slope), _lib.ptr(residual),
                                              ctypes.c_float(scale), 0 if accumulate_into is None else 1,
                                              ctypes.c_float(post_div), _lib.ptr(y), _lib.stream_ptr(x.device))
        _lib.check(rc, "conv1d_forward")
        return y
