"""Drop-ins for the VITS layer modules on the inference path, bound to libtts_b200.so.

Each class keeps the reference constructor signature, attribute names and ``state_dict`` keys (the torch
sub-modules are parameter containers only -- their ``forward`` is never called) and the reference
``forward`` signature for the inference direction:

  TextEncoder                  <- TTS/tts/layers/vits/networks.py:29-100
  ResidualCouplingBlocks       <- TTS/tts/layers/vits/networks.py:169-232   (reverse=True)
  StochasticDurationPredictor  <- TTS/tts/layers/vits/stochastic_duration_predictor.py:150-294 (reverse=True)
  ResidualCouplingBlocks       <- ... :223-227 (reverse=False, no log-det: the voice-conversion direction)
  PosteriorEncoder             <- TTS/tts/layers/vits/networks.py:235-288   (voice conversion)
  DurationPredictor            <- TTS/tts/layers/glow_tts/duration_predictor.py:22-69 (VitsArgs.use_sdp=False)

Training-only calls (SDP forward / likelihoods) raise NotImplementedError: this package is the inference hot path.
"""
import ctypes
import math

import torch
from torch import nn

from . import _lib


def _host(t):
    return None if t is None else t.detach().to(torch.float32).cpu().contiguous()


def _wb(m):
    """[weight, bias] of a conv container as host fp32 (weight norm folded by torch's parametrization)."""
    return [_host(m.weight), _host(m.bias)]


def _ln(n):
    """[gamma, beta] of a LayerNorm container as flat host fp32 vectors."""
    return [_host(n.gamma.reshape(-1)), _host(n.beta.reshape(-1))]


class EngineModule(nn.Module):
    """Owns one C-ABI handle built lazily from the module's parameters (and rebuilt after
    ``.to()`` / ``load_state_dict``).  Call ``repack()`` after editing weights in place."""

    _destroy = None  # name of the b200tts_*_destroy symbol

    def __init__(self):
        super().__init__()
        self._handle = None
        self._handle_device = None
        self._register_load_state_dict_pre_hook(lambda *a, **k: self._drop_handle())

    def _drop_handle(self):
        h = self.__dict__.get("_handle", None)
        if h is not None:
            getattr(_lib.lib(), self._destroy)(h)
        self._handle = None

    def repack(self):
        self._drop_handle()
        for m in self.children():
            if isinstance(m, EngineModule):
                m.repack()

    def __del__(self):
        try:
            self._drop_handle()
        except Exception:  # pragma: no cover
            pass

    def _apply(self, fn, *a, **kw):
        self._drop_handle()
        return super()._apply(fn, *a, **kw)

    def _create(self, device):  # -> ctypes.c_void_p
        raise NotImplementedError

    def handle(self, device):
        if self._handle is None or self._handle_device != device:
            self._drop_handle()
            with torch.cuda.device(device):
                self._handle = self._create(device)
            self._handle_device = device
        return self._handle

    @staticmethod
    def _make(create_name, cfg, tensors):
        arr = (ctypes.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])
        out = ctypes.c_void_p()
        rc = getattr(_lib.lib(), create_name)(ctypes.byref(cfg), arr, len(tensors), ctypes.byref(out))
        _lib.check(rc, create_name)
        return out


# ----------------------------------------------------------------------------- containers
class LayerNorm2(nn.Module):
    """Parameters of TTS/tts/layers/generic/normalization.py:31-53."""

    def __init__(self, channels, eps=1e-5):
        super().__init__()
        self.channels, self.eps = channels, eps
        self.gamma = nn.Parameter(torch.ones(channels))
        self.beta = nn.Parameter(torch.zeros(channels))


class WN(nn.Module):
    """Parameters of TTS/tts/layers/generic/wavenet.py:38-92 (weight-normed in/res_skip/cond layers)."""

    def __init__(self, in_channels, hidden_channels, kernel_size, dilation_rate, num_layers, c_in_channels=0,
                 dropout_p=0, weight_norm=True):
        super().__init__()
        assert kernel_size % 2 == 1 and hidden_channels % 2 == 0
        wn = torch.nn.utils.parametrizations.weight_norm if weight_norm else (lambda m, name="weight": m)
        self.in_channels, self.hidden_channels, self.kernel_size = in_channels, hidden_channels, kernel_size
        self.dilation_rate, self.num_layers, self.c_in_channels = dilation_rate, num_layers, c_in_channels
        self.in_layers = nn.ModuleList()
        self.res_skip_layers = nn.ModuleList()
        if c_in_channels > 0:
            self.cond_layer = wn(nn.Conv1d(c_in_channels, 2 * hidden_channels * num_layers, 1), name="weight")
        for i in range(num_layers):
            d = dilation_rate ** i
            cin = in_channels if i == 0 else hidden_channels
            self.in_layers.append(wn(nn.Conv1d(cin, 2 * hidden_channels, kernel_size, dilation=d,
                                               padding=int((kernel_size * d - d) / 2)), name="weight"))
            rs = 2 * hidden_channels if i < num_layers - 1 else hidden_channels
            self.res_skip_layers.append(wn(nn.Conv1d(hidden_channels, rs, 1), name="weight"))

    def ordered_weights(self):
        out = []
        if self.c_in_channels > 0:
            out += _wb(self.cond_layer)
        for a, b in zip(self.in_layers, self.res_skip_layers):
            out += _wb(a) + _wb(b)
        return out


class ResidualCouplingBlock(nn.Module):
    """Parameters of TTS/tts/layers/vits/networks.py:103-136."""

    def __init__(self, channels, hidden_channels, kernel_size, dilation_rate, num_layers, dropout_p=0,
                 cond_channels=0, mean_only=False):
        assert channels % 2 == 0, "channels should be divisible by 2"
        super().__init__()
        self.half_channels, self.mean_only = channels // 2, mean_only
        self.pre = nn.Conv1d(self.half_channels, hidden_channels, 1)
        self.enc = WN(hidden_channels, hidden_channels, kernel_size, dilation_rate, num_layers,
                      dropout_p=dropout_p, c_in_channels=cond_channels)
        self.post = nn.Conv1d(hidden_channels, self.half_channels * (2 - mean_only), 1)
        self.post.weight.data.zero_()
        self.post.bias.data.zero_()


class ResidualCouplingBlocks(EngineModule):
    _destroy = "b200tts_flow_destroy"

    def __init__(self, channels, hidden_channels, kernel_size, dilation_rate, num_layers, num_flows=4,
                 cond_channels=0):
        super().__init__()
        self.channels, self.hidden_channels, self.kernel_size = channels, hidden_channels, kernel_size
        self.dilation_rate, self.num_layers, self.num_flows = dilation_rate, num_layers, num_flows
        self.cond_channels = cond_channels
        self.flows = nn.ModuleList([
            ResidualCouplingBlock(channels, hidden_channels, kernel_size, dilation_rate, num_layers,
                                  cond_channels=cond_channels, mean_only=True) for _ in range(num_flows)])

    def _create(self, device, forward_direction=False):
        cfg = _lib.FlowConfigC(self.channels, self.hidden_channels, self.kernel_size, self.dilation_rate,
                               self.num_layers, self.num_flows, self.cond_channels)
        tensors = []
        for f in self.flows:
            tensors += _wb(f.pre) + f.enc.ordered_weights() + _wb(f.post)
        return self._make("b200tts_flow_create_forward" if forward_direction else "b200tts_flow_create", cfg, tensors)

    def _drop_forward_handle(self):
        h = self.__dict__.get("_handle_fwd", None)
        if h is not None:
            _lib.lib().b200tts_flow_destroy(h)
        self._handle_fwd = None

    def _drop_handle(self):
        """Both directions (weights changed: _apply / load_state_dict hook / repack / __del__)."""
        self._drop_reverse_handle()
        self._drop_forward_handle()

    def _drop_reverse_handle(self):
        EngineModule._drop_handle(self)

    def handle(self, device):
        # the two directions own separate handles: (re)creating one must not destroy the other (voice conversion
        # calls forward then reverse on every utterance)
        if self._handle is None or self._handle_device != device:
            self._drop_reverse_handle()
            with torch.cuda.device(device):
                self._handle = self._create(device)
            self._handle_device = device
        return self._handle

    def _forward_handle(self, device):
        if self.__dict__.get("_handle_fwd", None) is None or self._handle_fwd_device != device:
            self._drop_forward_handle()
            with torch.cuda.device(device):
                self._handle_fwd = self._create(device, forward_direction=True)
            self._handle_fwd_device = device
        return self._handle_fwd

    @torch.no_grad()
    def forward(self, x, x_mask, g=None, reverse=False, lengths=None):
        """x [B,C,T], x_mask [B,1,T], g [B,cond,1] -> z [B,C,T]   (networks.py:214-232).
        ``lengths`` (optional int [B] = the row sums of x_mask): padded frames are neither computed nor read; frames
        below a row's length are bit-identical to the dense call and the result is masked (zero) beyond it, as the
        reference's per-layer masking leaves it.
        reverse=True is the synthesis direction; reverse=False the posterior->prior direction used by voice
        conversion (the per-block log-determinant the reference discards at :226 is not computed)."""
        _lib.require_cuda(x, "x")
        if self.cond_channels > 0 and g is None:
            raise ValueError("tts_b200.ResidualCouplingBlocks: cond_channels > 0 but g is None")
        b, c, t_in = x.shape
        # everything in the flow is re-masked after each layer, so zero-masked extra frames are exact; padding T to
        # a multiple of 4 keeps activation rows 16-byte aligned for the tensor-core kernel's cp.async staging
        t = (t_in + 3) // 4 * 4
        z = torch.zeros((b, c, t), dtype=torch.float32, device=x.device)
        z[:, :, :t_in] = x
        mask = torch.zeros((b, 1, t), dtype=torch.float32, device=x.device)
        mask[:, :, :t_in] = x_mask
        gl = None if self.cond_channels == 0 else g.to(torch.float32).contiguous()
        h = self.handle(z.device) if reverse else self._forward_handle(z.device)
        L = _lib.lib()
        with torch.cuda.device(z.device):
            ws = _lib.workspace(z.device, L.b200tts_flow_workspace_bytes(h, b, t), "flow")
            if lengths is None:
                rc = L.b200tts_flow_reverse(h, _lib.ptr(z), _lib.ptr(mask), _lib.ptr(gl), b, t, _lib.ptr(ws),
                                            ctypes.c_size_t(ws.numel()), _lib.stream_ptr(z.device))
            else:
                lens = lengths.to(device=z.device, dtype=torch.int32).contiguous()
                rc = L.b200tts_flow_reverse_ragged(h, _lib.ptr(z), _lib.ptr(mask), _lib.ptr(gl), _lib.ptr(lens), b, t,
                                                   _lib.ptr(ws), ctypes.c_size_t(ws.numel()), _lib.stream_ptr(z.device))
        _lib.check(rc, "flow_reverse" if reverse else "flow_forward")
        if lengths is not None:
            z = z * mask         # rows keep their input values past their end in the ragged schedule: the reference has zeros
        if self.num_flows % 2:  # the channel flips are folded into the packed weights; an odd count leaves one over
            z = torch.flip(z, [1])
        return z if t == t_in else z[:, :, :t_in].contiguous()


class PosteriorEncoder(EngineModule):
    """TTS/tts/layers/vits/networks.py:235-288 (voice conversion / the encoder half of training)."""

    _destroy = "b200tts_posterior_destroy"

    def __init__(self, in_channels, out_channels, hidden_channels, kernel_size, dilation_rate, num_layers,
                 cond_channels=0):
        super().__init__()
        self.in_channels, self.out_channels, self.hidden_channels = in_channels, out_channels, hidden_channels
        self.kernel_size, self.dilation_rate, self.num_layers = kernel_size, dilation_rate, num_layers
        self.cond_channels = int(cond_channels or 0)
        self.pre = nn.Conv1d(in_channels, hidden_channels, 1)
        self.enc = WN(hidden_channels, hidden_channels, kernel_size, dilation_rate, num_layers,
                      c_in_channels=cond_channels)
        self.proj = nn.Conv1d(hidden_channels, out_channels * 2, 1)

    def _create(self, device):
        cfg = _lib.PosteriorConfigC(self.in_channels, self.out_channels, self.hidden_channels, self.kernel_size,
                                    self.dilation_rate, self.num_layers, self.cond_channels)
        return self._make("b200tts_posterior_create", cfg, _wb(self.pre) + self.enc.ordered_weights() + _wb(self.proj))

    @torch.no_grad()
    def forward(self, x, x_lengths, g=None, noise=None):
        """x [B,C,T] (linear spectrogram), x_lengths [B], g [B,cond,1] -> (z, mean, log_scale, x_mask)
        (networks.py:275-288).  ``noise`` [B,out,T] may be supplied; by default it is drawn on the device like
        the reference's ``torch.randn_like(mean)``."""
        _lib.require_cuda(x, "x")
        dev = x.device
        b, _, t_in = x.shape
        t = (t_in + 3) // 4 * 4            # 16-byte aligned rows for the tensor-core kernel (extra frames are masked)
        xs = torch.zeros((b, self.in_channels, t), dtype=torch.float32, device=dev)
        xs[:, :, :t_in] = x
        lens = x_lengths.to(dev)
        mask = (torch.arange(t, device=dev)[None, :] < lens[:, None]).to(torch.float32).unsqueeze(1).contiguous()
        if noise is None:
            noise = torch.randn((b, self.out_channels, t_in), dtype=torch.float32, device=dev)
        ns = torch.zeros((b, self.out_channels, t), dtype=torch.float32, device=dev)
        ns[:, :, :t_in] = noise.to(device=dev, dtype=torch.float32)
        if self.cond_channels > 0 and g is None:
            raise ValueError("tts_b200.PosteriorEncoder: cond_channels > 0 but g is None")
        gl = None if self.cond_channels == 0 else g.to(torch.float32).reshape(b, self.cond_channels).contiguous()
        z = torch.empty((b, self.out_channels, t), dtype=torch.float32, device=dev)
        stats = torch.empty((b, 2 * self.out_channels, t), dtype=torch.float32, device=dev)
        h = self.handle(dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            ws = _lib.workspace(dev, L.b200tts_posterior_workspace_bytes(h, b, t), "posterior")
            rc = L.b200tts_posterior_forward(h, _lib.ptr(xs), _lib.ptr(mask), _lib.ptr(gl), _lib.ptr(ns), b, t,
                                             _lib.ptr(z), _lib.ptr(stats), _lib.ptr(ws), ctypes.c_size_t(ws.numel()),
                                             _lib.stream_ptr(dev))
        _lib.check(rc, "posterior_forward")
        o = self.out_channels
        return (z[:, :, :t_in].contiguous(), stats[:, :o, :t_in].contiguous(), stats[:, o:, :t_in].contiguous(),
                mask[:, :, :t_in].contiguous())


class _LayerNorm1(nn.Module):
    """Parameters of TTS/tts/layers/generic/normalization.py:5-28 (gamma/beta shaped [1,C,1], eps 1e-4)."""

    def __init__(self, channels, eps=1e-4):
        super().__init__()
        self.channels, self.eps = channels, eps
        self.gamma = nn.Parameter(torch.ones(1, channels, 1) * 0.1)
        self.beta = nn.Parameter(torch.zeros(1, channels, 1))


class DurationPredictor(EngineModule):
    """TTS/tts/layers/glow_tts/duration_predictor.py:22-69 -- the deterministic predictor VITS builds when
    ``use_sdp=False`` (vits.py:646-654): conv-relu-LN-(dropout) x2 -> 1x1 projection to log-durations."""

    _destroy = "b200tts_duration_predictor_destroy"

    def __init__(self, in_channels, hidden_channels, kernel_size, dropout_p, cond_channels=None,
                 language_emb_dim=None):
        super().__init__()
        self._lang = int(language_emb_dim or 0)
        self._cond = int(cond_channels or 0)
        self._in = in_channels
        cin = in_channels + self._lang
        self.in_channels, self.filter_channels, self.kernel_size = cin, hidden_channels, kernel_size
        self.conv_1 = nn.Conv1d(cin, hidden_channels, kernel_size, padding=kernel_size // 2)
        self.norm_1 = _LayerNorm1(hidden_channels)
        self.conv_2 = nn.Conv1d(hidden_channels, hidden_channels, kernel_size, padding=kernel_size // 2)
        self.norm_2 = _LayerNorm1(hidden_channels)
        self.proj = nn.Conv1d(hidden_channels, 1, 1)
        if self._cond:
            self.cond = nn.Conv1d(self._cond, cin, 1)
        if self._lang:
            self.cond_lang = nn.Conv1d(self._lang, cin, 1)

    def ordered_weights(self):
        out = _wb(self.conv_1) + _ln(self.norm_1) + _wb(self.conv_2) + _ln(self.norm_2) + _wb(self.proj)
        if self._cond:
            out += _wb(self.cond)
        if self._lang:
            out += _wb(self.cond_lang)
        return out

    def _create(self, device):
        cfg = _lib.DurationPredictorConfigC(self._in, self.filter_channels, self.kernel_size, self._cond, self._lang)
        return self._make("b200tts_duration_predictor_create", cfg, self.ordered_weights())

    @torch.no_grad()
    def forward(self, x, x_mask, g=None, lang_emb=None):
        """x [B,C,T], x_mask [B,1,T], g [B,cond,1], lang_emb [B,L,1] -> log-durations [B,1,T]."""
        _lib.require_cuda(x, "x")
        dev = x.device
        x = x.to(torch.float32).contiguous()
        b, cin, t = x.shape
        if cin != self.in_channels:
            raise ValueError(f"tts_b200.DurationPredictor: expected {self.in_channels} input channels, got {cin}")
        mask = x_mask.to(torch.float32).expand(b, 1, t).contiguous()
        gl = g.to(torch.float32).reshape(b, self._cond).contiguous() if (self._cond and g is not None) else None
        ll = lang_emb.to(torch.float32).reshape(b, self._lang).contiguous() \
            if (self._lang and lang_emb is not None) else None
        logw = torch.empty((b, 1, t), dtype=torch.float32, device=dev)
        h = self.handle(dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            ws = _lib.workspace(dev, L.b200tts_duration_predictor_workspace_bytes(h, b, t), "duration_predictor")
            rc = L.b200tts_duration_predictor_forward(h, _lib.ptr(x), _lib.ptr(mask), _lib.ptr(gl), _lib.ptr(ll), b, t,
                                                      _lib.ptr(logw), _lib.ptr(ws), ctypes.c_size_t(ws.numel()),
                                                      _lib.stream_ptr(dev))
        _lib.check(rc, "duration_predictor_forward")
        return logw


# ----------------------------------------------------------------------------- text encoder
class _Attention(nn.Module):
    """Parameters of RelativePositionMultiHeadAttention (glow_tts/transformer.py:58-107)."""

    def __init__(self, channels, out_channels, num_heads, rel_attn_window_size=None, heads_share=True):
        super().__init__()
        assert channels % num_heads == 0
        self.k_channels = channels // num_heads
        self.conv_q = nn.Conv1d(channels, channels, 1)
        self.conv_k = nn.Conv1d(channels, channels, 1)
        self.conv_v = nn.Conv1d(channels, channels, 1)
        self.conv_o = nn.Conv1d(channels, out_channels, 1)
        if rel_attn_window_size is not None:
            n = 1 if heads_share else num_heads
            std = self.k_channels ** -0.5
            self.emb_rel_k = nn.Parameter(torch.randn(n, rel_attn_window_size * 2 + 1, self.k_channels) * std)
            self.emb_rel_v = nn.Parameter(torch.randn(n, rel_attn_window_size * 2 + 1, self.k_channels) * std)
        nn.init.xavier_uniform_(self.conv_q.weight)
        nn.init.xavier_uniform_(self.conv_k.weight)
        nn.init.xavier_uniform_(self.conv_v.weight)


class _FFN(nn.Module):
    def __init__(self, in_channels, out_channels, hidden_channels, kernel_size):
        super().__init__()
        self.conv_1 = nn.Conv1d(in_channels, hidden_channels, kernel_size)
        self.conv_2 = nn.Conv1d(hidden_channels, out_channels, kernel_size)


class RelativePositionTransformer(nn.Module):
    """Parameters of glow_tts/transformer.py:343-409 with in == hidden == out channels: layer_norm_type "2" and a
    relative window (the VITS text encoder) or "1" without one (Glow-TTS)."""

    def __init__(self, in_channels, out_channels, hidden_channels, hidden_channels_ffn, num_heads, num_layers,
                 kernel_size=1, dropout_p=0.0, rel_attn_window_size=None, input_length=None, layer_norm_type="1"):
        super().__init__()
        if layer_norm_type not in ("1", "2") or in_channels != hidden_channels or out_channels != hidden_channels:
            raise NotImplementedError("tts_b200: the transformer is built with in = hidden = out channels and "
                                      "layer_norm_type '1' or '2'")
        norm = _LayerNorm1 if layer_norm_type == "1" else LayerNorm2
        self.rel_attn_window_size = rel_attn_window_size
        self.attn_layers = nn.ModuleList()
        self.norm_layers_1 = nn.ModuleList()
        self.ffn_layers = nn.ModuleList()
        self.norm_layers_2 = nn.ModuleList()
        for _ in range(num_layers):
            self.attn_layers.append(_Attention(hidden_channels, hidden_channels, num_heads, rel_attn_window_size))
            self.norm_layers_1.append(norm(hidden_channels))
            self.ffn_layers.append(_FFN(hidden_channels, hidden_channels, hidden_channels_ffn, kernel_size))
            self.norm_layers_2.append(norm(hidden_channels))

    def ordered_weights(self):
        out = []
        for a, n1, f, n2 in zip(self.attn_layers, self.norm_layers_1, self.ffn_layers, self.norm_layers_2):
            if self.rel_attn_window_size is not None:
                if a.emb_rel_k.shape[0] != 1:
                    raise NotImplementedError("tts_b200: heads_share=False is not built")
                out += [_host(a.emb_rel_k), _host(a.emb_rel_v)]
            out += _wb(a.conv_q) + _wb(a.conv_k) + _wb(a.conv_v) + _wb(a.conv_o) + _ln(n1)
            out += _wb(f.conv_1) + _wb(f.conv_2) + _ln(n2)
        return out


class TextEncoder(EngineModule):
    _destroy = "b200tts_text_encoder_destroy"

    def __init__(self, n_vocab, out_channels, hidden_channels, hidden_channels_ffn, num_heads, num_layers,
                 kernel_size, dropout_p, language_emb_dim=None):
        super().__init__()
        self.out_channels, self.hidden_channels = out_channels, hidden_channels
        self._cfg = dict(n_vocab=n_vocab, out_channels=out_channels, hidden_channels=hidden_channels,
                         hidden_channels_ffn=hidden_channels_ffn, num_heads=num_heads, num_layers=num_layers,
                         kernel_size=kernel_size, language_emb_dim=int(language_emb_dim or 0))
        self.emb = nn.Embedding(n_vocab, hidden_channels)
        nn.init.normal_(self.emb.weight, 0.0, hidden_channels ** -0.5)
        c = hidden_channels + int(language_emb_dim or 0)
        self.encoder = RelativePositionTransformer(c, c, c, hidden_channels_ffn, num_heads, num_layers, kernel_size,
                                                   dropout_p, rel_attn_window_size=4, layer_norm_type="2")
        self.proj = nn.Conv1d(c, out_channels * 2, 1)

    def _create(self, device):
        c = self._cfg
        cfg = _lib.TextEncoderConfigC(c["n_vocab"], c["out_channels"], c["hidden_channels"],
                                      c["hidden_channels_ffn"], c["num_heads"], c["num_layers"], c["kernel_size"],
                                      self.encoder.rel_attn_window_size, c["language_emb_dim"])
        tensors = [_host(self.emb.weight)] + self.encoder.ordered_weights() + _wb(self.proj)
        return self._make("b200tts_text_encoder_create", cfg, tensors)

    @torch.no_grad()
    def forward(self, x, x_lengths, lang_emb=None):
        """x int64 [B,T], x_lengths [B] -> (x [B,C,T], m [B,out,T], logs [B,out,T], x_mask [B,1,T])
        (networks.py:80-100).  m and logs are views of one [B,2*out,T] tensor."""
        out, stats, mask = self.forward_stats(x, x_lengths, lang_emb)
        return out, stats[:, :self.out_channels], stats[:, self.out_channels:], mask

    @torch.no_grad()
    def forward_stats(self, x, x_lengths, lang_emb=None):
        """Same as forward but returns the packed statistics tensor [B, 2*out, T] (= cat(m, logs))."""
        _lib.require_cuda(x, "x")
        assert x.shape[0] == x_lengths.shape[0]
        dev = x.device
        tok = x.to(torch.int64).contiguous()
        lens = x_lengths.to(device=dev, dtype=torch.int64).contiguous()
        b, t = tok.shape
        ldim = self._cfg["language_emb_dim"]
        if (ldim > 0) != (lang_emb is not None):
            raise ValueError("tts_b200.TextEncoder: lang_emb does not match language_emb_dim")
        le = None if lang_emb is None else lang_emb.to(torch.float32).reshape(b, ldim).contiguous()
        c = self.hidden_channels + ldim
        out = torch.empty((b, c, t), dtype=torch.float32, device=dev)
        stats = torch.empty((b, 2 * self.out_channels, t), dtype=torch.float32, device=dev)
        mask = torch.empty((b, 1, t), dtype=torch.float32, device=dev)
        h = self.handle(dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            ws = _lib.workspace(dev, L.b200tts_text_encoder_workspace_bytes(h, b, t), "text_encoder")
            rc = L.b200tts_text_encoder_forward(h, _lib.ptr(tok), _lib.ptr(lens), _lib.ptr(le), b, t, _lib.ptr(out),
                                                _lib.ptr(stats), _lib.ptr(mask), _lib.ptr(ws),
                                                ctypes.c_size_t(ws.numel()), _lib.stream_ptr(dev))
        _lib.check(rc, "text_encoder_forward")
        return out, stats, mask


# ----------------------------------------------------------------------------- stochastic duration predictor
class DilatedDepthSeparableConv(nn.Module):
    """Parameters of stochastic_duration_predictor.py:11-44."""

    def __init__(self, channels, kernel_size, num_layers, dropout_p=0.0):
        super().__init__()
        self.num_layers = num_layers
        self.convs_sep, self.convs_1x1 = nn.ModuleList(), nn.ModuleList()
        self.norms_1, self.norms_2 = nn.ModuleList(), nn.ModuleList()
        for i in range(num_layers):
            d = kernel_size ** i
            self.convs_sep.append(nn.Conv1d(channels, channels, kernel_size, groups=channels, dilation=d,
                                            padding=(kernel_size * d - d) // 2))
            self.convs_1x1.append(nn.Conv1d(channels, channels, 1))
            self.norms_1.append(LayerNorm2(channels))
            self.norms_2.append(LayerNorm2(channels))

    def ordered_weights(self):
        out = []
        for s, c, n1, n2 in zip(self.convs_sep, self.convs_1x1, self.norms_1, self.norms_2):
            out += _wb(s) + _wb(c) + [_host(n1.gamma), _host(n1.beta), _host(n2.gamma), _host(n2.beta)]
        return out


class ElementwiseAffine(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.translation = nn.Parameter(torch.zeros(channels, 1))
        self.log_scale = nn.Parameter(torch.zeros(channels, 1))


class ConvFlow(nn.Module):
    """Parameters of stochastic_duration_predictor.py:100-118."""

    def __init__(self, in_channels, hidden_channels, kernel_size, num_layers, num_bins=10, tail_bound=5.0):
        super().__init__()
        self.num_bins, self.tail_bound, self.hidden_channels = num_bins, tail_bound, hidden_channels
        self.half_channels = in_channels // 2
        self.pre = nn.Conv1d(self.half_channels, hidden_channels, 1)
        self.convs = DilatedDepthSeparableConv(hidden_channels, kernel_size, num_layers, dropout_p=0.0)
        self.proj = nn.Conv1d(hidden_channels, self.half_channels * (num_bins * 3 - 1), 1)
        self.proj.weight.data.zero_()
        self.proj.bias.data.zero_()


class StochasticDurationPredictor(EngineModule):
    _destroy = "b200tts_sdp_destroy"

    def __init__(self, in_channels, hidden_channels, kernel_size, dropout_p, num_flows=4, cond_channels=0,
                 language_emb_dim=0):
        super().__init__()
        language_emb_dim = int(language_emb_dim or 0)
        cond_channels = int(cond_channels or 0)
        self._cfg = dict(in_channels=in_channels, hidden_channels=hidden_channels, kernel_size=kernel_size,
                         num_flows=num_flows, cond_channels=cond_channels, language_emb_dim=language_emb_dim)
        cin = in_channels + language_emb_dim
        self.pre = nn.Conv1d(cin, hidden_channels, 1)
        self.convs = DilatedDepthSeparableConv(hidden_channels, kernel_size, num_layers=3, dropout_p=dropout_p)
        self.proj = nn.Conv1d(hidden_channels, hidden_channels, 1)
        self.flows = nn.ModuleList([ElementwiseAffine(2)] +
                                   [ConvFlow(2, hidden_channels, kernel_size, num_layers=3) for _ in range(num_flows)])
        self.post_pre = nn.Conv1d(1, hidden_channels, 1)
        self.post_convs = DilatedDepthSeparableConv(hidden_channels, kernel_size, num_layers=3, dropout_p=dropout_p)
        self.post_proj = nn.Conv1d(hidden_channels, hidden_channels, 1)
        self.post_flows = nn.ModuleList([ElementwiseAffine(2)] +
                                        [ConvFlow(2, hidden_channels, kernel_size, num_layers=3)
                                         for _ in range(num_flows)])
        if cond_channels != 0:
            self.cond = nn.Conv1d(cond_channels, hidden_channels, 1)
        if language_emb_dim != 0:
            self.cond_lang = nn.Conv1d(language_emb_dim, hidden_channels, 1)

    def _create(self, device):
        c = self._cfg
        cfg = _lib.SdpConfigC(c["in_channels"], c["hidden_channels"], c["kernel_size"], c["num_flows"],
                              c["cond_channels"], c["language_emb_dim"], self.flows[1].num_bins,
                              float(self.flows[1].tail_bound))
        tensors = _wb(self.pre)
        if c["cond_channels"]:
            tensors += _wb(self.cond)
        if c["language_emb_dim"]:
            tensors += _wb(self.cond_lang)
        tensors += self.convs.ordered_weights() + _wb(self.proj)
        tensors += [_host(self.flows[0].translation), _host(self.flows[0].log_scale)]
        for f in list(self.flows)[1:]:
            tensors += _wb(f.pre) + f.convs.ordered_weights() + _wb(f.proj)
        return self._make("b200tts_sdp_create", cfg, tensors)

    @torch.no_grad()
    def forward(self, x, x_mask, dr=None, g=None, lang_emb=None, reverse=False, noise_scale=1.0, noise=None):
        """reverse=True: x [B,C,T], x_mask [B,1,T], g [B,cond,1] -> logw [B,1,T]
        (stochastic_duration_predictor.py:222-239,285-294).  ``noise`` [B,2,T] may be supplied; by default it
        is drawn exactly like the reference: torch.randn on the CPU generator, then moved (:287)."""
        if not reverse:
            raise NotImplementedError("tts_b200: the SDP is implemented for inference (reverse=True) only")
        _lib.require_cuda(x, "x")
        dev = x.device
        x = x.to(torch.float32).contiguous()
        b, cin, t = x.shape
        c = self._cfg
        if c["language_emb_dim"]:
            if lang_emb is None:
                raise ValueError("tts_b200.StochasticDurationPredictor: lang_emb required")
        mask = x_mask.to(torch.float32).expand(b, 1, t).contiguous()
        if noise is None:
            noise = torch.randn(b, 2, t)
        noise = noise.to(device=dev, dtype=torch.float32).contiguous()
        gl = None
        if c["cond_channels"] and g is not None:
            gl = g.to(torch.float32).reshape(b, c["cond_channels"]).contiguous()
        ll = None
        if c["language_emb_dim"] and lang_emb is not None:
            ll = lang_emb.to(torch.float32).reshape(b, c["language_emb_dim"]).contiguous()
        logw = torch.empty((b, 1, t), dtype=torch.float32, device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        h = self.handle(dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            ws = _lib.workspace(dev, L.b200tts_sdp_workspace_bytes(h, b, t), "sdp")
            rc = L.b200tts_sdp_reverse(h, _lib.ptr(x), _lib.ptr(mask), _lib.ptr(noise), _lib.ptr(gl), _lib.ptr(ll),
                                       ctypes.c_float(noise_scale), b, t, _lib.ptr(logw), _lib.ptr(flag),
                                       _lib.ptr(ws), ctypes.c_size_t(ws.numel()), _lib.stream_ptr(dev))
        _lib.check(rc, "sdp_reverse")
        self.last_error_flag = flag  # checked lazily by Vits.inference at its host sync point
        return logw


def durations_to_path(logw, x_mask, length_scale, err_flag=None):
    """Stage 1 of vits.py:1140-1146 on the device: returns (w_ceil [B,1,T], cum [B,T], y_lengths int64 [B],
    meta int64 [2] = {max(y_lengths), err_flag}) -- one D2H read of ``meta`` is the path's only host sync."""
    dev = logw.device
    b, _, t = logw.shape
    logw = logw.to(torch.float32).contiguous()
    mask = x_mask.to(torch.float32).expand(b, 1, t).contiguous()
    w_ceil = torch.empty((b, 1, t), dtype=torch.float32, device=dev)
    cum = torch.empty((b, t), dtype=torch.float32, device=dev)
    y_lengths = torch.empty((b,), dtype=torch.int64, device=dev)
    meta = torch.empty((2,), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().b200tts_durations(_lib.ptr(logw), _lib.ptr(mask), ctypes.c_float(length_scale), b, t,
                                          _lib.ptr(w_ceil), _lib.ptr(cum), _lib.ptr(y_lengths), _lib.ptr(err_flag),
                                          _lib.ptr(meta), _lib.stream_ptr(dev))
    _lib.check(rc, "durations")
    return w_ceil, cum, y_lengths, meta


def expand_prior(cum, x_mask, y_lengths, stats, noise, noise_scale, t_dec, want_attn=True):
    """Stage 2 of vits.py:1147-1155: (attn [B,Tx,Ty], m_p, logs_p, z_p [B,C,Ty], y_mask [B,1,Ty])."""
    dev = cum.device
    b, tx = cum.shape
    c = stats.shape[1] // 2
    stats = stats.contiguous()
    mask = x_mask.to(torch.float32).reshape(b, tx).contiguous()
    noise = noise.to(device=dev, dtype=torch.float32).contiguous()
    attn = torch.empty((b, tx, t_dec), dtype=torch.float32, device=dev) if want_attn else None
    m_p = torch.empty((b, c, t_dec), dtype=torch.float32, device=dev)
    logs_p = torch.empty_like(m_p)
    z_p = torch.empty_like(m_p)
    y_mask = torch.empty((b, 1, t_dec), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().b200tts_expand_prior(_lib.ptr(cum), _lib.ptr(mask), _lib.ptr(y_lengths), _lib.ptr(stats),
                                             _lib.ptr(noise), ctypes.c_float(noise_scale), b, tx, t_dec, c,
                                             _lib.ptr(attn), _lib.ptr(m_p), _lib.ptr(logs_p), _lib.ptr(z_p),
                                             _lib.ptr(y_mask), _lib.stream_ptr(dev))
    _lib.check(rc, "expand_prior")
    return attn, m_p, logs_p, z_p, y_mask


def upsample_linear(z, scale_factor):
    """F.interpolate(z, scale_factor=[f], mode="linear") on the device (vits.py:952): [B,C,T] -> [B,C,floor(T*f)]."""
    _lib.require_cuda(z, "z")
    z = z.to(torch.float32).contiguous()
    b, c, t = z.shape
    t_out = int(math.floor(t * float(scale_factor)))
    out = torch.empty((b, c, t_out), dtype=torch.float32, device=z.device)
    with torch.cuda.device(z.device):
        rc = _lib.lib().b200tts_upsample_linear(_lib.ptr(z), b * c, t, ctypes.c_float(scale_factor), _lib.ptr(out), t_out,
                                                _lib.stream_ptr(z.device))
    _lib.check(rc, "upsample_linear")
    return out
