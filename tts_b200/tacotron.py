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
from dataclasses import dataclass

from torch import nn

from . import _lib
from .layers import _host
from .tacotron2 import (Tacotron2Config, _check_config, _DynamicConvolutionAttention, _OriginalAttention, _Prenet,
                        _TacotronBase)


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


# ----------------------------------------------------------------------------- model
class Tacotron(_TacotronBase):
    """Tacotron text -> spectrogram synthesiser, inference path on sm_90a kernels."""

    _destroy = "b200tts_tacotron_destroy"
    _model = "tacotron"
    _width = 256
    _extra_steps = 1      # the reference stops once t > max_decoder_steps

    def __init__(self, config, ap=None, tokenizer=None, speaker_manager=None):
        super().__init__()
        _check_config(config, self._model, self._width)
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

    # ------------------------------------------------------------------ packing
    def _create(self, device):
        d = self.decoder
        cfg = _lib.TacotronConfigC(self.num_chars, self.decoder_output_dim, self.out_channels, d.r_init,
                                   int(self.memory_size), int(self.attention_type == "dynamic_convolution"),
                                   int(bool(self.location_attn)), int(self.attention_norm == "softmax"),
                                   int(self.prenet_type == "bn"), int(bool(self.prenet_dropout)))
        t = [_host(self.embedding.weight)]
        for lin in self.encoder.prenet.linear_layers:
            t += [_host(lin.linear_layer.weight), _host(lin.linear_layer.bias)]
        t += _cbhg_weights(self.encoder.cbhg.cbhg)
        for lin in d.prenet.linear_layers:
            t += [_host(lin.linear_layer.weight), _host(lin.linear_layer.bias)]
            if self.prenet_type == "bn":
                bn = lin.batch_normalization
                t += [_host(bn.weight), _host(bn.bias), _host(bn.running_mean), _host(bn.running_var)]
        t += self._cell(d.attention_rnn)
        t += self._attention_weights(d.attention)
        t += [_host(d.project_to_decoder_in.weight), _host(d.project_to_decoder_in.bias)]
        for cell in d.decoder_rnns:
            t += self._cell(cell)
        t += [_host(d.proj_to_mel.weight), _host(d.proj_to_mel.bias), _host(d.stopnet.linear.weight),
              _host(d.stopnet.linear.bias)]
        t += _cbhg_weights(self.postnet.cbhg)
        t += [_host(self.last_linear.weight), _host(self.last_linear.bias)]
        return self._make("b200tts_tacotron_create", cfg, t)

    def _check_call(self):
        super()._check_call()
        if self.training:
            raise NotImplementedError("tts_b200: Tacotron inference in training mode (the encoder prenet's dropout) "
                                      "is not built; call eval() first")
