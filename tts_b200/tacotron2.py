"""Drop-in for the inference path of TTS.tts.models.tacotron2.Tacotron2 (TTS/tts/models/tacotron2.py:21-300), with the
model-side fields of TacotronConfig / Tacotron2Config (TTS/tts/configs/tacotron_config.py, tacotron2_config.py), on
sm_90a kernels.

``inference`` runs in one library handle: the encoder (embedding, conv + BatchNorm blocks, bidirectional LSTM), the
attention decoder loop on the device (CUDA graph chunks of steps, one small host read per chunk) and the postnet.
``model_outputs`` ``[B, T, 80]`` feeds ``tts_b200.vocoder.vocoder_input`` and the vocoders directly.

Kept surface: ``Tacotron2(config, ap, tokenizer, speaker_manager)``, ``init_from_config``, ``inference(text,
aux_input)``, ``load_checkpoint(config, path, eval)`` (with the reference's resolution of ``r``) and the reference
``state_dict`` keys, ``coarse_decoder.*`` included (double decoder consistency: the coarse decoder's weights load but
do not run at inference, as in the reference).

Differences from the reference, on purpose:

1. Batched, per row.  The reference cannot run more than one row (its stop test raises for B > 1, and its encoder and
   attention have no masks at inference).  Here ``aux_input["x_lengths"]`` gives each row's length (default: the
   nonzero tokens), and row b equals the reference's ``inference(text[b:b+1, :x_lengths[b]])``: the one-row stop rule
   (a row never stops at step 0), zeros past each row in every output.  The output dict adds ``model_outputs_len``,
   the mel frames per row.
2. Random draws.  With ``prenet_dropout_at_inference`` the reference draws the prenet dropout masks with two generator
   calls per step.  Here they are drawn in bulk on the device before the loop, or taken from the keyword argument
   ``draws`` (an addition to the reference signature): ``{"dropout": [B, max_decoder_steps, 2, 256] bool or uint8}``,
   nonzero keeps a unit (doubled).

Out of scope (construction raises ``NotImplementedError``): graves attention, attention windowing, forward attention
and the transition agent, GST and Capacitron, speaker embeddings and d-vectors, the bidirectional decoder, encoder /
decoder widths other than 512, the Tacotron (1) model (``tts_b200.tacotron.Tacotron``), and training (``forward``).
"""
import ctypes
from dataclasses import dataclass
from typing import List

import torch
from scipy.stats import betabinom
from torch import nn

from . import _lib
from .layers import EngineModule, _host
from .overflow import _ConfigBase, _format_aux_input, _Linear

CHUNK_STEPS = 32      # decoder steps per CUDA graph replay (one host read per chunk)
PRENET_DIM = 256


@dataclass
class Tacotron2Config(_ConfigBase):
    """The model-side fields of TTS/tts/configs/tacotron2_config.py (TacotronConfig) with the reference defaults."""
    model: str = "tacotron2"
    use_gst: bool = False
    gst: dict = None
    gst_style_input: str = None
    use_capacitron_vae: bool = False
    capacitron_vae: dict = None
    num_speakers: int = 1
    num_chars: int = 0
    r: int = 2
    gradual_training: List[List[int]] = None
    memory_size: int = -1
    prenet_type: str = "original"
    prenet_dropout: bool = True
    prenet_dropout_at_inference: bool = False
    stopnet: bool = True
    separate_stopnet: bool = True
    stopnet_pos_weight: float = 0.2
    max_decoder_steps: int = 10000
    encoder_in_features: int = 512
    decoder_in_features: int = 512
    decoder_output_dim: int = 80
    out_channels: int = 80
    attention_type: str = "original"
    attention_heads: int = None
    attention_norm: str = "sigmoid"
    attention_win: bool = False
    windowing: bool = False
    use_forward_attn: bool = False
    forward_attn_mask: bool = False
    transition_agent: bool = False
    location_attn: bool = True
    bidirectional_decoder: bool = False
    double_decoder_consistency: bool = False
    ddc_r: int = 6
    speakers_file: str = None
    use_speaker_embedding: bool = False
    speaker_embedding_dim: int = 512
    use_d_vector_file: bool = False
    d_vector_file: str = False
    d_vector_dim: int = None


# ----------------------------------------------------------------------------- parameter containers
class _ConvBNBlock(nn.Module):
    """Parameters of TTS/tts/layers/tacotron/tacotron2.py:11-44."""

    def __init__(self, in_channels, out_channels, kernel_size=5):
        super().__init__()
        self.convolution1d = nn.Conv1d(in_channels, out_channels, kernel_size, padding=(kernel_size - 1) // 2)
        self.batch_normalization = nn.BatchNorm1d(out_channels, momentum=0.1, eps=1e-5)


class _Encoder(nn.Module):
    """Parameters of tacotron2.py:73-92."""

    def __init__(self, channels=512):
        super().__init__()
        self.convolutions = nn.ModuleList([_ConvBNBlock(channels, channels) for _ in range(3)])
        self.lstm = nn.LSTM(channels, channels // 2, num_layers=1, batch_first=True, bias=True, bidirectional=True)


class _LinearBN(nn.Module):
    """Parameters of common_layers.py:28-60."""

    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.linear_layer = nn.Linear(in_features, out_features, bias=bias)
        self.batch_normalization = nn.BatchNorm1d(out_features, momentum=0.1, eps=1e-5)


class _Prenet(nn.Module):
    """Parameters of common_layers.py:63-119 (bias=False, as the Tacotron2 decoder builds it; Tacotron's with bias)."""

    def __init__(self, in_features, prenet_type, out_features, bias=False):
        super().__init__()
        ins = [in_features] + out_features[:-1]
        layer = _LinearBN if prenet_type == "bn" else _Linear
        self.linear_layers = nn.ModuleList([layer(i, o, bias=bias) for i, o in zip(ins, out_features)])


class _LocationLayer(nn.Module):
    """Parameters of attentions.py:9-37."""

    def __init__(self, attention_dim, n_filters=32, kernel_size=31):
        super().__init__()
        self.location_conv1d = nn.Conv1d(2, n_filters, kernel_size, padding=(kernel_size - 1) // 2, bias=False)
        self.location_dense = _Linear(n_filters, attention_dim, bias=False)


class _OriginalAttention(nn.Module):
    """Parameters of attentions.py:127-196 (no transition agent)."""

    def __init__(self, query_dim, embedding_dim, attention_dim, location_attention):
        super().__init__()
        self.query_layer = _Linear(query_dim, attention_dim, bias=False)
        self.inputs_layer = _Linear(embedding_dim, attention_dim, bias=False)
        self.v = _Linear(attention_dim, 1, bias=True)
        if location_attention:
            self.location_layer = _LocationLayer(attention_dim)


class _DynamicConvolutionAttention(nn.Module):
    """Parameters of attentions.py:323-389 (MonotonicDynamicConvolutionAttention, 8 filters of 21 taps, prior 11)."""

    def __init__(self, query_dim, attention_dim, filters=8, kernel=21, prior_len=11, alpha=0.1, beta=0.9):
        super().__init__()
        self.query_layer = nn.Linear(query_dim, attention_dim)
        self.key_layer = nn.Linear(attention_dim, filters * kernel, bias=False)
        self.static_filter_conv = nn.Conv1d(1, filters, kernel, padding=(kernel - 1) // 2, bias=False)
        self.static_filter_layer = nn.Linear(filters, attention_dim, bias=False)
        self.dynamic_filter_layer = nn.Linear(filters, attention_dim)
        self.v = nn.Linear(attention_dim, 1, bias=False)
        prior = betabinom.pmf(range(prior_len), prior_len - 1, alpha, beta)
        self.register_buffer("prior", torch.FloatTensor(prior).flip(0))


class _Decoder(nn.Module):
    """Parameters of tacotron2.py:116-209 (query / decoder RNN 1024, attention 128, prenet 256)."""

    def __init__(self, in_channels, frame_channels, r, attn_type, prenet_type, location_attn):
        super().__init__()
        self.frame_channels, self.r_init, self.r = frame_channels, r, r
        self.prenet = _Prenet(frame_channels, prenet_type, [PRENET_DIM, PRENET_DIM])
        self.attention_rnn = nn.LSTMCell(PRENET_DIM + in_channels, 1024, bias=True)
        if attn_type == "original":
            self.attention = _OriginalAttention(1024, in_channels, 128, location_attn)
        else:
            self.attention = _DynamicConvolutionAttention(1024, 128)
        self.decoder_rnn = nn.LSTMCell(1024 + in_channels, 1024, bias=True)
        self.linear_projection = _Linear(1024 + in_channels, frame_channels * r)
        self.stopnet = nn.Sequential(nn.Dropout(0.1), _Linear(1024 + frame_channels * r, 1, bias=True))

    def set_r(self, new_r):
        self.r = new_r


class _Postnet(nn.Module):
    """Parameters of tacotron2.py:47-70."""

    def __init__(self, channels, num_convs=5):
        super().__init__()
        chans = [channels] + [512] * (num_convs - 1) + [channels]
        self.convolutions = nn.ModuleList([_ConvBNBlock(chans[i], chans[i + 1]) for i in range(num_convs)])


# config.model -> the class name and where the other model of the family is
_MODELS = {"tacotron": ("Tacotron", "Tacotron2 is tts_b200.tacotron2.Tacotron2"),
           "tacotron2": ("Tacotron2", "the Tacotron 1 model is tts_b200.tacotron.Tacotron")}


def _check_config(cfg, model, width):
    """NotImplementedError for every option this drop-in of ``model`` ("tacotron" / "tacotron2", encoder and decoder
    widths ``width``) does not build."""
    name, other = _MODELS[model]

    def no(what):
        raise NotImplementedError(f"tts_b200: {name} with {what} is not built")

    if getattr(cfg, "model", model) != model:
        no(f"model {cfg.model!r} (only {name}; {other})")
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
    if cfg.encoder_in_features != width or cfg.decoder_in_features != width:
        no(f"encoder / decoder widths other than {width} (the reference's embedding is fixed at {width})")
    if cfg.prenet_type not in ("original", "bn"):
        no(f"prenet_type {cfg.prenet_type!r}")
    if cfg.attention_norm not in ("sigmoid", "softmax"):
        raise ValueError("Unknown value for attention norm type")


# ----------------------------------------------------------------------------- models
class _TacotronBase(EngineModule):
    """What Tacotron and Tacotron2 share: the inference driver over the library's encode / decode_loop / postnet calls,
    the attention's weight list, the config check, construction from a config and checkpoints.  A subclass sets
    ``_model`` (the C-ABI prefix and ``config.model``), ``_width`` (encoder output width) and ``_extra_steps``."""

    _model = None
    _width = None
    _extra_steps = 0      # decoder steps a row may run past max_decoder_steps

    @classmethod
    def init_from_config(cls, config, samples=None, verbose=True):  # pylint: disable=unused-argument
        """base_tacotron.py init_from_config without the host-side managers (built by the caller)."""
        return cls(config)

    def _check_call(self):
        _check_config(self, self._model, self._width)

    @staticmethod
    def _cell(m):
        return [_host(m.weight_ih), _host(m.weight_hh), _host(m.bias_ih), _host(m.bias_hh)]

    def _attention_weights(self, a):
        """The attention's tensors in the order TacoAttention::init reads them."""
        if self.attention_type == "dynamic_convolution":
            return [_host(a.prior), _host(a.query_layer.weight), _host(a.query_layer.bias), _host(a.key_layer.weight),
                    _host(a.static_filter_conv.weight), _host(a.static_filter_layer.weight),
                    _host(a.dynamic_filter_layer.weight), _host(a.dynamic_filter_layer.bias), _host(a.v.weight)]
        t = [_host(a.query_layer.linear_layer.weight), _host(a.inputs_layer.linear_layer.weight),
             _host(a.v.linear_layer.weight), _host(a.v.linear_layer.bias)]
        if self.location_attn:
            t += [_host(a.location_layer.location_conv1d.weight),
                  _host(a.location_layer.location_dense.linear_layer.weight)]
        return t

    def _dropout_active(self):
        return bool(self.prenet_dropout) and (self.training or bool(self.prenet_dropout_at_inference))

    # ------------------------------------------------------------------ inference
    @torch.no_grad()
    def inference(self, text, aux_input=None, *, draws=None):
        """text int64 [B, T] (CUDA) -> dict(model_outputs [B, T_out, out_channels], decoder_outputs [B, T_out, C],
        alignments [B, T_dec, T], stop_tokens [B, T_dec, 1], model_outputs_len [B]).  ``draws`` (optional): the prenet
        dropout masks, see the module docstring.  One host read per chunk of 32 decoder steps drives the loop."""
        self._check_call()
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
        steps_cap = max_steps + self._extra_steps
        r, c = int(self.decoder.r), self.decoder_output_dim
        if not 1 <= r <= self.decoder.r_init:
            raise ValueError(f"tts_b200: r must be in [1, {self.decoder.r_init}], got {r}")
        drop = None
        if self._dropout_active():
            drop = (draws or {}).get("dropout", None)
            if drop is None:
                drop = torch.empty((b, steps_cap, 2, PRENET_DIM), dtype=torch.uint8, device=dev).bernoulli_(0.5)
            else:
                if drop.shape[0] != b or drop.shape[1] < steps_cap or tuple(drop.shape[2:]) != (2, PRENET_DIM):
                    raise ValueError(f"tts_b200: draws['dropout'] must be [{b}, >= {steps_cap}, 2, {PRENET_DIM}], "
                                     f"got {tuple(drop.shape)}")
                drop = drop[:, :steps_cap].to(dev, torch.uint8).contiguous()
        f32 = dict(dtype=torch.float32, device=dev)
        enc = torch.empty((b, tt, self._width), **f32)
        dec = torch.empty((b, steps_cap * r, c), **f32)
        stop = torch.empty((b, steps_cap), **f32)
        align = torch.empty((b, steps_cap, tt), **f32)
        steps = (ctypes.c_int32 * b)()
        h = self.handle(dev)
        L, m = _lib.lib(), self._model
        s = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            # the encoder and the loop; the postnet's scratch is sized below from the frames the loop produced
            ws = _lib.workspace(dev, getattr(L, f"b200tts_{m}_workspace_bytes")(h, b, tt, 0), m)
            wsp, wsn = _lib.ptr(ws), ctypes.c_size_t(ws.numel())
            _lib.check(getattr(L, f"b200tts_{m}_encode")(h, _lib.ptr(tok), _lib.ptr(lens), b, tt, _lib.ptr(enc), wsp,
                                                         wsn, s), f"{m}_encode")
            _lib.check(getattr(L, f"b200tts_{m}_decode_loop")(h, _lib.ptr(lens), _lib.ptr(enc), b, tt, r, max_steps,
                                                              _lib.ptr(drop), CHUNK_STEPS, _lib.ptr(dec),
                                                              _lib.ptr(stop), _lib.ptr(align), steps, wsp, wsn, s),
                       f"{m}_decode_loop")
            n_steps = torch.tensor(list(steps), dtype=torch.int32)
            t_dec = int(n_steps.max())
            frames = (n_steps * r).to(dev)
            out = torch.empty((b, t_dec * r, self.out_channels), **f32)
            ws = _lib.workspace(dev, getattr(L, f"b200tts_{m}_workspace_bytes")(h, b, tt, t_dec * r), m)
            wsp, wsn = _lib.ptr(ws), ctypes.c_size_t(ws.numel())
            _lib.check(getattr(L, f"b200tts_{m}_postnet")(h, _lib.ptr(dec), _lib.ptr(frames), b, t_dec * r,
                                                          steps_cap * r, _lib.ptr(out), wsp, wsn, s), f"{m}_postnet")
        return {"model_outputs": out, "decoder_outputs": dec[:, :t_dec * r], "alignments": align[:, :t_dec],
                "stop_tokens": stop[:, :t_dec].unsqueeze(-1),
                "model_outputs_len": (n_steps * r).to(device=dev, dtype=x_lengths.dtype)}

    # ------------------------------------------------------------------ out of scope
    def forward(self, *args, **kwargs):
        raise NotImplementedError(f"tts_b200: {_MODELS[self._model][0]} implements inference only; training (forward) is out of scope")

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


class Tacotron2(_TacotronBase):
    """Tacotron2 text -> mel synthesiser, inference path on sm_90a kernels."""

    _destroy = "b200tts_tacotron2_destroy"
    _model = "tacotron2"
    _width = 512

    def __init__(self, config, ap=None, tokenizer=None, speaker_manager=None):
        super().__init__()
        _check_config(config, self._model, self._width)
        self.config, self.ap, self.tokenizer, self.speaker_manager = config, ap, tokenizer, speaker_manager
        for key in config:
            setattr(self, key, config[key])
        if tokenizer is not None:   # BaseTTS._set_model_args
            self.num_chars = tokenizer.characters.num_chars
        self.decoder_output_dim = self.out_channels
        self.embedding = nn.Embedding(self.num_chars, 512, padding_idx=0)
        self.encoder = _Encoder(self.encoder_in_features)
        self.decoder = _Decoder(self.decoder_in_features, self.out_channels, self.r, self.attention_type,
                                self.prenet_type, self.location_attn)
        self.postnet = _Postnet(self.out_channels)
        if self.double_decoder_consistency:
            self.coarse_decoder = _Decoder(self.decoder_in_features, self.out_channels, self.ddc_r,
                                           self.attention_type, self.prenet_type, self.location_attn)

    # ------------------------------------------------------------------ packing
    def _create(self, device):
        d = self.decoder
        cfg = _lib.Tacotron2ConfigC(self.num_chars, self.out_channels, d.r_init,
                                    int(self.attention_type == "dynamic_convolution"), int(bool(self.location_attn)),
                                    int(self.attention_norm == "softmax"), int(self.prenet_type == "bn"),
                                    int(bool(self.prenet_dropout)))
        t = [_host(self.embedding.weight)]
        for blk in list(self.encoder.convolutions):
            t += self._conv_bn(blk)
        for sfx in ("", "_reverse"):
            t += [_host(getattr(self.encoder.lstm, f"{n}_l0{sfx}")) for n in ("weight_ih", "weight_hh", "bias_ih",
                                                                              "bias_hh")]
        for lin in d.prenet.linear_layers:
            t += [_host(lin.linear_layer.weight)]
            if self.prenet_type == "bn":
                bn = lin.batch_normalization
                t += [_host(bn.weight), _host(bn.bias), _host(bn.running_mean), _host(bn.running_var)]
        t += self._cell(d.attention_rnn)
        t += self._attention_weights(d.attention)
        t += self._cell(d.decoder_rnn)
        t += [_host(d.linear_projection.linear_layer.weight), _host(d.linear_projection.linear_layer.bias),
              _host(d.stopnet[1].linear_layer.weight), _host(d.stopnet[1].linear_layer.bias)]
        for blk in self.postnet.convolutions:
            t += self._conv_bn(blk)
        return self._make("b200tts_tacotron2_create", cfg, t)

    @staticmethod
    def _conv_bn(blk):
        bn = blk.batch_normalization
        return [_host(blk.convolution1d.weight), _host(blk.convolution1d.bias), _host(bn.weight), _host(bn.bias),
                _host(bn.running_mean), _host(bn.running_var)]
