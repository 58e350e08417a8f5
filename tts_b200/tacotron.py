"""Drop-in for the inference path of TTS.tts.models.tacotron.Tacotron (TTS/tts/models/tacotron.py:218-271), with the
model-side fields of TacotronConfig (TTS/tts/configs/tacotron_config.py), on sm_90a kernels.

``inference`` runs in one library handle: the encoder (embedding, prenet, CBHG with its persistent bidirectional GRU),
the GRU attention decoder loop on the device (CUDA graph chunks of steps, one small host read per chunk) and the
postnet (CBHG and last_linear).  With ``out_channels == decoder_output_dim`` (80 for a mel vocoder) ``model_outputs``
``[B, T, out_channels]`` feeds ``tts_b200.vocoder.vocoder_input`` and the vocoders directly.

Kept surface: ``Tacotron(config, ap, tokenizer, speaker_manager)``, ``init_from_config``, ``inference(text,
aux_input)``, ``load_checkpoint(config, path, eval)`` (with the reference's resolution of ``r``) and the reference
``state_dict`` keys, BatchNorm ``num_batches_tracked`` and ``coarse_decoder.*`` included (double decoder consistency:
the coarse decoder's weights load but do not run at inference, as in the reference).

Differences from the reference, on purpose:

1. Batched, per row.  The reference runs one row (its stop test reads one attention weight).  Here
   ``aux_input["x_lengths"]`` gives each row's length (default: the nonzero tokens), and row b equals the reference's
   ``inference(text[b:b+1, :x_lengths[b]])``: every conv sees zero padding at the row's end, the backward GRUs start at
   the row's last token or frame, the stop rule reads the row's own length and last token, and every output is zero
   past the row.  The output dict adds ``model_outputs_len``, the frames per row.
2. Random draws.  With ``prenet_dropout_at_inference`` the reference draws the decoder prenet's dropout masks with two
   generator calls per step.  Here they are drawn in bulk on the device before the loop, or taken from the keyword
   argument ``draws`` (an addition to the reference signature): ``{"dropout": [B, max_decoder_steps + 1, 2, 256] bool
   or uint8}`` (layer 1 reads the first 128 of its 256), nonzero keeps a unit (doubled).

Out of scope (construction or the call raises ``NotImplementedError``): GST and Capacitron, speaker embeddings and
d-vectors, graves attention, windowing, forward attention and the transition agent, the bidirectional decoder,
encoder / decoder widths other than 256, inference in training mode (the encoder prenet's dropout), and training
(``forward``).  Also not built: streaming and 16-bit precision.
A linear output reaches audio through ``tts_b200.audio.AudioProcessor.inv_spectrogram`` (Griffin-Lim on the device).
"""
import ctypes
from dataclasses import dataclass

import torch
from torch import nn

from . import _lib
from .layers import EngineModule, _host
from .overflow import _format_aux_input
from .tacotron2 import CHUNK_STEPS, Tacotron2Config, _DynamicConvolutionAttention, _OriginalAttention, _Prenet

PRENET_DIM = 256


@dataclass
class TacotronConfig(Tacotron2Config):
    """The model-side fields of TTS/tts/configs/tacotron_config.py (TacotronConfig) with the reference defaults; the
    same fields as Tacotron2Config, which the reference derives from it."""
    model: str = "tacotron"
    encoder_in_features: int = 256
    decoder_in_features: int = 256
    out_channels: int = 513


# ----------------------------------------------------------------------------- parameter containers
class _BatchNormConv1d(nn.Module):
    """Parameters of TTS/tts/layers/tacotron/tacotron.py:11-58 (no conv bias, BatchNorm eps 1e-3)."""

    def __init__(self, in_channels, out_channels, kernel_size):
        super().__init__()
        self.conv1d = nn.Conv1d(in_channels, out_channels, kernel_size, bias=False)
        self.bn = nn.BatchNorm1d(out_channels, momentum=0.99, eps=1e-3)


class _Highway(nn.Module):
    """Parameters of tacotron.py:61-91."""

    def __init__(self, features):
        super().__init__()
        self.H = nn.Linear(features, features)
        self.T = nn.Linear(features, features)


class _CBHG(nn.Module):
    """Parameters of tacotron.py:94-188 (bank 128 channels, 4 highways of 128, GRU 128)."""

    def __init__(self, in_features, K, conv_projections):
        super().__init__()
        self.conv1d_banks = nn.ModuleList([_BatchNormConv1d(in_features, 128, k) for k in range(1, K + 1)])
        ins = [K * 128] + conv_projections[:-1]
        self.conv1d_projections = nn.ModuleList([_BatchNormConv1d(i, o, 3) for i, o in zip(ins, conv_projections)])
        if conv_projections[-1] != 128:
            self.pre_highway = nn.Linear(conv_projections[-1], 128, bias=False)
        self.highways = nn.ModuleList([_Highway(128) for _ in range(4)])
        self.gru = nn.GRU(128, 128, 1, batch_first=True, bidirectional=True)


class _CBHGHolder(nn.Module):
    """EncoderCBHG / PostCBHG (tacotron.py:191-246): a module holding ``cbhg``."""

    def __init__(self, in_features, K, conv_projections):
        super().__init__()
        self.cbhg = _CBHG(in_features, K, conv_projections)


class _Encoder(nn.Module):
    """Parameters of tacotron.py:210-229."""

    def __init__(self, in_features):
        super().__init__()
        self.prenet = _Prenet(in_features, "original", [256, 128], bias=True)
        self.cbhg = _CBHGHolder(128, 16, [128, 128])


class _StopNet(nn.Module):
    """Parameters of tacotron.py:488-503."""

    def __init__(self, in_features):
        super().__init__()
        self.dropout = nn.Dropout(0.1)
        self.linear = nn.Linear(in_features, 1)


class _Decoder(nn.Module):
    """Parameters of tacotron.py:249-334 (query / decoder RNN 256, attention 128, prenet [256, 128] with bias)."""

    def __init__(self, in_channels, frame_channels, r, memory_size, attn_type, prenet_type, location_attn):
        super().__init__()
        self.frame_channels, self.r_init, self.r = frame_channels, r, r
        self.use_memory_queue = memory_size > 0
        self.memory_size = memory_size if memory_size > 0 else r
        prenet_dim = frame_channels * self.memory_size if self.use_memory_queue else frame_channels
        self.prenet = _Prenet(prenet_dim, prenet_type, [256, 128], bias=True)
        self.attention_rnn = nn.GRUCell(in_channels + 128, 256)
        if attn_type == "original":
            self.attention = _OriginalAttention(256, in_channels, 128, location_attn)
        else:
            self.attention = _DynamicConvolutionAttention(256, 128)
        self.project_to_decoder_in = nn.Linear(256 + in_channels, 256)
        self.decoder_rnns = nn.ModuleList([nn.GRUCell(256, 256) for _ in range(2)])
        self.proj_to_mel = nn.Linear(256, frame_channels * self.r_init)
        self.stopnet = _StopNet(256 + frame_channels * self.r_init)

    def set_r(self, new_r):
        self.r = new_r


class TacotronConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("n_vocab", "frame_channels", "out_channels", "r_init", "memory_size",
                                            "attention_type", "location_attn", "attention_norm", "prenet_bn",
                                            "prenet_dropout")]


def _declare(L):
    if getattr(L, "_tacotron_declared", False):
        return
    vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    L.b200tts_tacotron_create.restype = ci
    L.b200tts_tacotron_create.argtypes = [ctypes.POINTER(TacotronConfigC), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
    L.b200tts_tacotron_destroy.restype = None
    L.b200tts_tacotron_destroy.argtypes = [vp]
    L.b200tts_tacotron_workspace_bytes.restype = sz
    L.b200tts_tacotron_workspace_bytes.argtypes = [vp, ci, ci, ci]
    L.b200tts_tacotron_encode.restype = ci
    L.b200tts_tacotron_encode.argtypes = [vp, vp, vp, ci, ci, vp, vp, sz, vp]
    L.b200tts_tacotron_decode_loop.restype = ci
    L.b200tts_tacotron_decode_loop.argtypes = [vp, vp, vp, ci, ci, ci, ci, vp, ci, vp, vp, vp, vp, vp, sz, vp]
    L.b200tts_tacotron_postnet.restype = ci
    L.b200tts_tacotron_postnet.argtypes = [vp, vp, vp, ci, ci, ci, vp, vp, sz, vp]
    L._tacotron_declared = True


def _check_config(cfg):
    """NotImplementedError for every option this drop-in does not build."""
    def no(what):
        raise NotImplementedError(f"tts_b200: Tacotron with {what} is not built")

    if getattr(cfg, "model", "tacotron") != "tacotron":
        no(f"model {cfg.model!r} (only Tacotron; Tacotron2 is tts_b200.tacotron2.Tacotron2)")
    if cfg.attention_type not in ("original", "dynamic_convolution"):
        no(f"attention_type {cfg.attention_type!r}")
    if cfg.attention_win or cfg.windowing:
        no("attention windowing")
    if cfg.use_forward_attn or cfg.forward_attn_mask or cfg.transition_agent:
        no("forward attention / the transition agent")
    if cfg.use_gst:
        no("global style tokens")
    if cfg.use_capacitron_vae:
        no("Capacitron")
    if cfg.num_speakers > 1 or cfg.use_speaker_embedding or cfg.use_d_vector_file:
        no("speaker embeddings / d-vectors")
    if cfg.bidirectional_decoder:
        no("the bidirectional decoder")
    if cfg.encoder_in_features != 256 or cfg.decoder_in_features != 256:
        no("encoder / decoder widths other than 256 (the reference's embedding is fixed at 256)")
    if cfg.prenet_type not in ("original", "bn"):
        no(f"prenet_type {cfg.prenet_type!r}")
    if cfg.attention_norm not in ("sigmoid", "softmax"):
        raise ValueError("Unknown value for attention norm type")


def _cbhg_weights(cb):
    t = []
    for blk in list(cb.conv1d_banks) + list(cb.conv1d_projections):
        t += [_host(blk.conv1d.weight), _host(blk.bn.weight), _host(blk.bn.bias), _host(blk.bn.running_mean),
              _host(blk.bn.running_var)]
    if hasattr(cb, "pre_highway"):
        t.append(_host(cb.pre_highway.weight))
    for hw in cb.highways:
        t += [_host(hw.H.weight), _host(hw.H.bias), _host(hw.T.weight), _host(hw.T.bias)]
    for sfx in ("", "_reverse"):
        t += [_host(getattr(cb.gru, f"{n}_l0{sfx}")) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return t


def _cell(m):
    return [_host(m.weight_ih), _host(m.weight_hh), _host(m.bias_ih), _host(m.bias_hh)]


# ----------------------------------------------------------------------------- model
class Tacotron(EngineModule):
    """Tacotron text -> spectrogram synthesiser, inference path on sm_90a kernels."""

    _destroy = "b200tts_tacotron_destroy"

    def __init__(self, config, ap=None, tokenizer=None, speaker_manager=None):
        super().__init__()
        _check_config(config)
        self.config, self.ap, self.tokenizer, self.speaker_manager = config, ap, tokenizer, speaker_manager
        for key in config:
            setattr(self, key, config[key])
        if tokenizer is not None:   # BaseTTS._set_model_args
            self.num_chars = tokenizer.characters.num_chars
        self.embedding = nn.Embedding(self.num_chars, 256, padding_idx=0)
        self.encoder = _Encoder(self.encoder_in_features)
        self.decoder = _Decoder(self.decoder_in_features, self.decoder_output_dim, self.r, self.memory_size,
                                self.attention_type, self.prenet_type, self.location_attn)
        self.postnet = _CBHGHolder(self.decoder_output_dim, 8, [256, self.decoder_output_dim])
        self.last_linear = nn.Linear(256, self.out_channels)
        if self.double_decoder_consistency:
            self.coarse_decoder = _Decoder(self.decoder_in_features, self.decoder_output_dim, self.ddc_r,
                                           self.memory_size, self.attention_type, self.prenet_type, self.location_attn)

    @classmethod
    def init_from_config(cls, config, samples=None, verbose=True):  # pylint: disable=unused-argument
        """base_tacotron.py init_from_config without the host-side managers (built by the caller)."""
        return cls(config)

    # ------------------------------------------------------------------ packing
    def _create(self, device):
        d = self.decoder
        dca = self.attention_type == "dynamic_convolution"
        cfg = TacotronConfigC(self.num_chars, self.decoder_output_dim, self.out_channels, d.r_init,
                              int(self.memory_size), int(dca), int(bool(self.location_attn)),
                              int(self.attention_norm == "softmax"), int(self.prenet_type == "bn"),
                              int(bool(self.prenet_dropout)))
        t = [_host(self.embedding.weight)]
        for lin in self.encoder.prenet.linear_layers:
            t += [_host(lin.linear_layer.weight), _host(lin.linear_layer.bias)]
        t += _cbhg_weights(self.encoder.cbhg.cbhg)
        for lin in d.prenet.linear_layers:
            t += [_host(lin.linear_layer.weight), _host(lin.linear_layer.bias)]
            if self.prenet_type == "bn":
                bn = lin.batch_normalization
                t += [_host(bn.weight), _host(bn.bias), _host(bn.running_mean), _host(bn.running_var)]
        t += _cell(d.attention_rnn)
        a = d.attention
        if dca:
            t += [_host(a.prior), _host(a.query_layer.weight), _host(a.query_layer.bias), _host(a.key_layer.weight),
                  _host(a.static_filter_conv.weight), _host(a.static_filter_layer.weight),
                  _host(a.dynamic_filter_layer.weight), _host(a.dynamic_filter_layer.bias), _host(a.v.weight)]
        else:
            t += [_host(a.query_layer.linear_layer.weight), _host(a.inputs_layer.linear_layer.weight),
                  _host(a.v.linear_layer.weight), _host(a.v.linear_layer.bias)]
            if self.location_attn:
                t += [_host(a.location_layer.location_conv1d.weight),
                      _host(a.location_layer.location_dense.linear_layer.weight)]
        t += [_host(d.project_to_decoder_in.weight), _host(d.project_to_decoder_in.bias)]
        for cell in d.decoder_rnns:
            t += _cell(cell)
        t += [_host(d.proj_to_mel.weight), _host(d.proj_to_mel.bias), _host(d.stopnet.linear.weight),
              _host(d.stopnet.linear.bias)]
        t += _cbhg_weights(self.postnet.cbhg)
        t += [_host(self.last_linear.weight), _host(self.last_linear.bias)]
        _declare(_lib.lib())
        return self._make("b200tts_tacotron_create", cfg, t)

    # ------------------------------------------------------------------ inference
    @torch.no_grad()
    def inference(self, text, aux_input=None, *, draws=None):
        """text int64 [B, T] (CUDA) -> dict(model_outputs [B, T_out, out_channels], decoder_outputs [B, T_out, C],
        alignments [B, T_dec, T], stop_tokens [B, T_dec, 1], model_outputs_len [B]).  ``draws`` (optional): the prenet
        dropout masks, see the module docstring.  One host read per chunk of 32 decoder steps drives the loop."""
        _check_config(self)
        if self.training:
            raise NotImplementedError("tts_b200: Tacotron inference in training mode (the encoder prenet's dropout) "
                                      "is not built; call eval() first")
        _lib.require_cuda(text, "text")
        dev = text.device
        tok = text.to(torch.int64).contiguous()
        b, tt = tok.shape
        if b == 0:
            raise ValueError("tts_b200: empty batch")
        aux = _format_aux_input({"x_lengths": torch.sum(text != 0, dim=1)}, aux_input)
        x_lengths = aux["x_lengths"]
        lens = x_lengths.to(device=dev, dtype=torch.int64).contiguous()
        if int(lens.min()) < 1 or int(lens.max()) > tt:
            raise ValueError(f"tts_b200: x_lengths must be in [1, {tt}]")
        max_steps = int(self.max_decoder_steps)
        if max_steps < 1:
            raise ValueError("tts_b200: max_decoder_steps must be >= 1")
        steps_cap = max_steps + 1   # the reference stops once t > max_decoder_steps
        r, c = int(self.decoder.r), self.decoder_output_dim
        if not 1 <= r <= self.decoder.r_init:
            raise ValueError(f"tts_b200: r must be in [1, {self.decoder.r_init}], got {r}")
        drop = None
        if bool(self.prenet_dropout) and bool(self.prenet_dropout_at_inference):
            drop = (draws or {}).get("dropout", None)
            if drop is None:
                drop = torch.empty((b, steps_cap, 2, PRENET_DIM), dtype=torch.uint8, device=dev).bernoulli_(0.5)
            else:
                if drop.shape[0] != b or drop.shape[1] < steps_cap or tuple(drop.shape[2:]) != (2, PRENET_DIM):
                    raise ValueError(f"tts_b200: draws['dropout'] must be [{b}, >= {steps_cap}, 2, {PRENET_DIM}], "
                                     f"got {tuple(drop.shape)}")
                drop = drop[:, :steps_cap].to(dev, torch.uint8).contiguous()
        f32 = dict(dtype=torch.float32, device=dev)
        enc = torch.empty((b, tt, 256), **f32)
        dec = torch.empty((b, steps_cap * r, c), **f32)
        stop = torch.empty((b, steps_cap), **f32)
        align = torch.empty((b, steps_cap, tt), **f32)
        steps = (ctypes.c_int32 * b)()
        h = self.handle(dev)
        L = _lib.lib()
        _declare(L)
        s = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            # the encoder and the loop; the postnet's scratch is sized below from the frames the loop produced
            ws = _lib.workspace(dev, L.b200tts_tacotron_workspace_bytes(h, b, tt, 0), "tacotron")
            wsp, wsn = _lib.ptr(ws), ctypes.c_size_t(ws.numel())
            _lib.check(L.b200tts_tacotron_encode(h, _lib.ptr(tok), _lib.ptr(lens), b, tt, _lib.ptr(enc), wsp, wsn, s),
                       "tacotron_encode")
            _lib.check(L.b200tts_tacotron_decode_loop(h, _lib.ptr(lens), _lib.ptr(enc), b, tt, r, max_steps,
                                                      _lib.ptr(drop), CHUNK_STEPS, _lib.ptr(dec), _lib.ptr(stop),
                                                      _lib.ptr(align), steps, wsp, wsn, s), "tacotron_decode_loop")
            n_steps = torch.tensor(list(steps), dtype=torch.int32)
            t_dec = int(n_steps.max())
            frames = (n_steps * r).to(dev)
            out = torch.empty((b, t_dec * r, self.out_channels), **f32)
            ws = _lib.workspace(dev, L.b200tts_tacotron_workspace_bytes(h, b, tt, t_dec * r), "tacotron")
            wsp, wsn = _lib.ptr(ws), ctypes.c_size_t(ws.numel())
            _lib.check(L.b200tts_tacotron_postnet(h, _lib.ptr(dec), _lib.ptr(frames), b, t_dec * r, steps_cap * r,
                                                  _lib.ptr(out), wsp, wsn, s), "tacotron_postnet")
        return {"model_outputs": out, "decoder_outputs": dec[:, :t_dec * r], "alignments": align[:, :t_dec],
                "stop_tokens": stop[:, :t_dec].unsqueeze(-1),
                "model_outputs_len": (n_steps * r).to(device=dev, dtype=x_lengths.dtype)}

    # ------------------------------------------------------------------ out of scope
    def forward(self, *args, **kwargs):
        raise NotImplementedError("tts_b200: Tacotron implements inference only; training (forward) is out of scope")

    # ------------------------------------------------------------------ checkpoints (base_tacotron.py:94-120)
    def load_checkpoint(self, config, checkpoint_path, eval=False, cache=False):  # pylint: disable=unused-argument, redefined-builtin
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        if "r" in state:
            self.decoder.set_r(state["r"])
        elif "config" in state:
            self.decoder.set_r(state["config"]["r"])
        else:
            self.decoder.set_r(config.r)
        self._drop_handle()
        if eval:
            self.eval()
            assert not self.training
