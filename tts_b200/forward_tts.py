"""Drop-in for the inference path of TTS.tts.models.forward_tts.ForwardTTS (TTS/tts/models/forward_tts.py:172-862) --
FastPitch, FastSpeech and FastSpeech2 -- and the model-side fields of their configs, on sm_90a kernels.

The whole of ``ForwardTTS.inference`` runs in one library handle: encoder, speaker add, duration / pitch / energy
predictors and durations on the exact FP32 FMA conv, then the expansion, positional encoding and FFTransformer decoder
on the 3xTF32 tensor-core convs and attention kernel.  Its ``[B, T', C]`` mel output feeds
``tts_b200.vocoder.vocoder_input`` and a HiFiGAN vocoder directly.

Unlike the reference, inference is batched: ``aux_input["x_lengths"]`` is honoured (all ``T`` tokens are valid when it
is absent) and row ``b`` equals the reference's single-utterance ``inference(x[b:b+1, :x_lengths[b]])``.  The reference
itself cannot batch (its ``x_lengths = torch.tensor(x.shape[1:2])``, :686, fails in ``nn.MultiheadAttention`` for
``B > 1``).  The one difference at ``B = 1``: an ``x_lengths[0] < T`` is honoured instead of ignored.

Kept surface: ``ForwardTTS(config, ap, tokenizer, speaker_manager)``, ``ForwardTTS.init_from_config``,
``inference(x, aux_input)`` -> the reference's 5-key dict plus ``durations`` and ``y_lengths``,
``load_checkpoint(config, path, eval)``, ``length_scale``, ``init_multispeaker`` and the reference ``state_dict`` keys
(``pos_encoder.pe`` and the training-only ``aligner.*`` included; the aligner is loaded and never run).  Built for
``encoder_type`` / ``decoder_type`` "fftransformer"; other types, training and ``forward`` raise
``NotImplementedError``.
"""
import copy
import ctypes
import math
from dataclasses import asdict, dataclass, field

import torch
from torch import nn

from . import _lib
from .layers import DurationPredictor, EngineModule, _host, _wb


# ----------------------------------------------------------------------------- configs
class _ConfigMixin:
    def __getitem__(self, k):
        return getattr(self, k)

    def __setitem__(self, k, v):
        setattr(self, k, v)

    def __contains__(self, k):
        return hasattr(self, k)

    def __iter__(self):
        return iter(asdict(self))

    def get(self, k, default=None):
        return getattr(self, k, default)


def _fft_params():
    return {"hidden_channels_ffn": 1024, "num_heads": 1, "num_layers": 6, "dropout_p": 0.1}


@dataclass
class ForwardTTSArgs(_ConfigMixin):
    """TTS/tts/models/forward_tts.py:22-169 with the reference defaults (``poisitonal_encoding_use_scale`` keeps the
    reference's spelling; like there, it has no effect)."""
    num_chars: int = None
    out_channels: int = 80
    hidden_channels: int = 384
    use_aligner: bool = True
    use_pitch: bool = True
    pitch_predictor_hidden_channels: int = 256
    pitch_predictor_kernel_size: int = 3
    pitch_predictor_dropout_p: float = 0.1
    pitch_embedding_kernel_size: int = 3
    use_energy: bool = False
    energy_predictor_hidden_channels: int = 256
    energy_predictor_kernel_size: int = 3
    energy_predictor_dropout_p: float = 0.1
    energy_embedding_kernel_size: int = 3
    duration_predictor_hidden_channels: int = 256
    duration_predictor_kernel_size: int = 3
    duration_predictor_dropout_p: float = 0.1
    positional_encoding: bool = True
    poisitonal_encoding_use_scale: bool = True
    length_scale: int = 1
    encoder_type: str = "fftransformer"
    encoder_params: dict = field(default_factory=_fft_params)
    decoder_type: str = "fftransformer"
    decoder_params: dict = field(default_factory=_fft_params)
    detach_duration_predictor: bool = False
    max_duration: int = 75
    num_speakers: int = 1
    use_speaker_embedding: bool = False
    speakers_file: str = None
    use_d_vector_file: bool = False
    d_vector_dim: int = None
    d_vector_file: str = None


@dataclass
class _ForwardTTSConfig(_ConfigMixin):
    """The model-side fields shared by fast_pitch_config.py, fast_speech_config.py, fastspeech2_config.py and
    speedy_speech_config.py, with their ``__post_init__`` (multi-speaker settings copied into ``model_args``)."""
    model: str = "forward_tts"
    base_model: str = "forward_tts"
    model_args: ForwardTTSArgs = field(default_factory=ForwardTTSArgs)
    num_speakers: int = 0
    speakers_file: str = None
    use_speaker_embedding: bool = False
    use_d_vector_file: bool = False
    d_vector_file: str = False
    d_vector_dim: int = 0

    def __post_init__(self):
        if self.num_speakers > 0:
            self.model_args.num_speakers = self.num_speakers
        if self.use_speaker_embedding:
            self.model_args.use_speaker_embedding = True
        if self.speakers_file:
            self.model_args.speakers_file = self.speakers_file
        if self.use_d_vector_file:
            self.model_args.use_d_vector_file = True
        if self.d_vector_dim is not None and self.d_vector_dim > 0:
            self.model_args.d_vector_dim = self.d_vector_dim
        if self.d_vector_file:
            self.model_args.d_vector_file = self.d_vector_file


@dataclass
class FastPitchConfig(_ForwardTTSConfig):
    """TTS/tts/configs/fast_pitch_config.py (model-side fields)."""
    model: str = "fast_pitch"


@dataclass
class FastSpeechConfig(_ForwardTTSConfig):
    """TTS/tts/configs/fast_speech_config.py (model-side fields): no pitch predictor."""
    model: str = "fast_speech"
    model_args: ForwardTTSArgs = field(default_factory=lambda: ForwardTTSArgs(use_pitch=False))


@dataclass
class FastSpeech2Config(_ForwardTTSConfig):
    """TTS/tts/configs/fastspeech2_config.py (model-side fields): pitch and energy predictors."""
    model: str = "fastspeech2"
    model_args: ForwardTTSArgs = field(default_factory=lambda: ForwardTTSArgs(use_pitch=True, use_energy=True))


Fastspeech2Config = FastSpeech2Config   # the reference's spelling (TTS/tts/configs/fastspeech2_config.py)


@dataclass
class SpeedySpeechConfig(_ForwardTTSConfig):
    """TTS/tts/configs/speedy_speech_config.py (model-side fields).  Its ``residual_conv_bn`` encoder and decoder are
    not built: ``ForwardTTS`` raises ``NotImplementedError`` for it."""
    model: str = "speedy_speech"
    model_args: ForwardTTSArgs = field(default_factory=lambda: ForwardTTSArgs(
        use_pitch=False, encoder_type="residual_conv_bn",
        encoder_params={"kernel_size": 4, "dilations": 4 * [1, 2, 4] + [1], "num_conv_blocks": 2, "num_res_blocks": 13},
        decoder_type="residual_conv_bn",
        decoder_params={"kernel_size": 4, "dilations": 4 * [1, 2, 4, 8] + [1], "num_conv_blocks": 2,
                        "num_res_blocks": 17},
        out_channels=80, hidden_channels=128, positional_encoding=True, detach_duration_predictor=True))


# ----------------------------------------------------------------------------- parameter containers
class _FFTransformer(nn.Module):
    """Parameters of TTS/tts/layers/generic/transformer.py:6-19 (kernel_size_fft 3)."""

    def __init__(self, in_out_channels, num_heads, hidden_channels_ffn=1024, kernel_size_fft=3, dropout_p=0.1):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(in_out_channels, num_heads, dropout=dropout_p)
        padding = (kernel_size_fft - 1) // 2
        self.conv1 = nn.Conv1d(in_out_channels, hidden_channels_ffn, kernel_size=kernel_size_fft, padding=padding)
        self.conv2 = nn.Conv1d(hidden_channels_ffn, in_out_channels, kernel_size=kernel_size_fft, padding=padding)
        self.norm1 = nn.LayerNorm(in_out_channels)
        self.norm2 = nn.LayerNorm(in_out_channels)

    def weights(self):
        a = self.self_attn
        return [_host(a.in_proj_weight), _host(a.in_proj_bias), _host(a.out_proj.weight), _host(a.out_proj.bias)] + \
            _wb(self.conv1) + _wb(self.conv2) + _wb(self.norm1) + _wb(self.norm2)


class _FFTransformerBlock(nn.Module):
    """Parameters of TTS/tts/layers/generic/transformer.py:38-52."""

    def __init__(self, in_out_channels, num_heads, hidden_channels_ffn, num_layers, dropout_p):
        super().__init__()
        self.fft_layers = nn.ModuleList([_FFTransformer(in_out_channels, num_heads, hidden_channels_ffn,
                                                        dropout_p=dropout_p) for _ in range(num_layers)])


def _check_type(kind, name):
    if name.lower() != "fftransformer":
        raise NotImplementedError(f"tts_b200.ForwardTTS: {kind}_type {name!r} is not built (fftransformer only)")


class _Encoder(nn.Module):
    """Parameters of TTS/tts/layers/feed_forward/encoder.py:76-152 for encoder_type "fftransformer"."""

    def __init__(self, in_hidden_channels, out_channels, encoder_type, encoder_params, c_in_channels=0):
        super().__init__()
        _check_type("encoder", encoder_type)
        assert in_hidden_channels == out_channels, \
            "[!] must be `in_channels` == `out_channels` when encoder type is 'fftransformer'"
        self.out_channels, self.in_channels, self.hidden_channels = out_channels, in_hidden_channels, in_hidden_channels
        self.encoder_type, self.c_in_channels = encoder_type, c_in_channels
        self.encoder = _FFTransformerBlock(in_hidden_channels, **encoder_params)


class _FFTransformerDecoder(nn.Module):
    """Parameters of TTS/tts/layers/feed_forward/decoder.py:94-115."""

    def __init__(self, in_channels, out_channels, params):
        super().__init__()
        self.transformer_block = _FFTransformerBlock(in_channels, **params)
        self.postnet = nn.Conv1d(in_channels, out_channels, 1)


class _Decoder(nn.Module):
    """Parameters of TTS/tts/layers/feed_forward/decoder.py:163-217 for decoder_type "fftransformer"."""

    def __init__(self, out_channels, in_hidden_channels, decoder_type, decoder_params):
        super().__init__()
        _check_type("decoder", decoder_type)
        self.decoder = _FFTransformerDecoder(in_hidden_channels, out_channels, decoder_params)


class _PositionalEncoding(nn.Module):
    """The ``pe`` buffer of TTS/tts/layers/generic/pos_encoding.py:18-36 (use_scale False, as ForwardTTS builds it)."""

    def __init__(self, channels, max_len=5000):
        super().__init__()
        if channels % 2 != 0:
            raise ValueError("Cannot use sin/cos positional encoding with "
                             "odd channels (got channels={:d})".format(channels))
        pe = torch.zeros(max_len, channels)
        position = torch.arange(0, max_len).unsqueeze(1)
        div_term = torch.pow(10000, torch.arange(0, channels, 2).float() / channels)
        pe[:, 0::2] = torch.sin(position.float() * div_term)
        pe[:, 1::2] = torch.cos(position.float() * div_term)
        self.register_buffer("pe", pe.unsqueeze(0).transpose(1, 2))
        self.channels = channels


class _AlignmentNetwork(nn.Module):
    """Parameters of TTS/tts/layers/generic/aligner.py:22-58 -- training only: loaded with the checkpoint, never run."""

    def __init__(self, in_query_channels=80, in_key_channels=512, attn_channels=80):
        super().__init__()
        self.key_layer = nn.Sequential(nn.Conv1d(in_key_channels, in_key_channels * 2, 3, padding=1), nn.ReLU(),
                                       nn.Conv1d(in_key_channels * 2, attn_channels, 1))
        self.query_layer = nn.Sequential(nn.Conv1d(in_query_channels, in_query_channels * 2, 3, padding=1), nn.ReLU(),
                                         nn.Conv1d(in_query_channels * 2, in_query_channels, 1), nn.ReLU(),
                                         nn.Conv1d(in_query_channels, attn_channels, 1))


# ----------------------------------------------------------------------------- model
class ForwardTTS(EngineModule):
    """FastPitch / FastSpeech / FastSpeech2 text -> mel synthesiser, inference path on sm_90a kernels."""

    _destroy = "b200tts_forward_tts_destroy"

    def __init__(self, config, ap=None, tokenizer=None, speaker_manager=None):
        super().__init__()
        self.config, self.ap, self.tokenizer, self.speaker_manager = config, ap, tokenizer, speaker_manager
        self.args = config.model_args if hasattr(config, "model_args") else config   # BaseTTS._set_model_args
        if tokenizer is not None:
            self.args.num_chars = tokenizer.characters.num_chars
        a = self.args
        self.init_multispeaker(config)
        self.max_duration, self.use_aligner = a.max_duration, a.use_aligner
        self.use_pitch, self.use_energy = a.use_pitch, a.use_energy
        self.binary_loss_weight = 0.0
        self.length_scale = float(a.length_scale) if isinstance(a.length_scale, int) else a.length_scale
        self.emb = nn.Embedding(a.num_chars, a.hidden_channels)
        self.encoder = _Encoder(a.hidden_channels, a.hidden_channels, a.encoder_type, a.encoder_params,
                                self.embedded_speaker_dim)
        if a.positional_encoding:
            self.pos_encoder = _PositionalEncoding(a.hidden_channels)
        self.decoder = _Decoder(a.out_channels, a.hidden_channels, a.decoder_type, a.decoder_params)
        self.duration_predictor = DurationPredictor(a.hidden_channels, a.duration_predictor_hidden_channels,
                                                    a.duration_predictor_kernel_size, a.duration_predictor_dropout_p)
        if a.use_pitch:
            self.pitch_predictor = DurationPredictor(a.hidden_channels, a.pitch_predictor_hidden_channels,
                                                     a.pitch_predictor_kernel_size, a.pitch_predictor_dropout_p)
            self.pitch_emb = nn.Conv1d(1, a.hidden_channels, kernel_size=a.pitch_embedding_kernel_size,
                                       padding=int((a.pitch_embedding_kernel_size - 1) / 2))
        if a.use_energy:
            self.energy_predictor = DurationPredictor(a.hidden_channels, a.energy_predictor_hidden_channels,
                                                      a.energy_predictor_kernel_size, a.energy_predictor_dropout_p)
            self.energy_emb = nn.Conv1d(1, a.hidden_channels, kernel_size=a.energy_embedding_kernel_size,
                                        padding=int((a.energy_embedding_kernel_size - 1) / 2))
        if a.use_aligner:
            self.aligner = _AlignmentNetwork(in_query_channels=a.out_channels, in_key_channels=a.hidden_channels)

    def init_multispeaker(self, config):
        """forward_tts.py:283-308."""
        self.embedded_speaker_dim = 0
        if self.speaker_manager is None and (config.use_d_vector_file or config.use_speaker_embedding):
            raise ValueError(" > SpeakerManager is not provided. You must provide the SpeakerManager before "
                             "initializing a multi-speaker model.")
        if self.speaker_manager is not None:
            self.num_speakers = self.speaker_manager.num_speakers
        if config.use_d_vector_file:
            self.embedded_speaker_dim = config.d_vector_dim
            if self.args.d_vector_dim != self.args.hidden_channels:
                self.proj_g = nn.Linear(in_features=self.args.d_vector_dim, out_features=self.args.hidden_channels)
        if config.use_speaker_embedding and not config.use_d_vector_file:
            self.emb_g = nn.Embedding(self.num_speakers, self.args.hidden_channels)
            nn.init.uniform_(self.emb_g.weight, -0.1, 0.1)

    @staticmethod
    def init_from_config(config, samples=None):  # pylint: disable=unused-argument
        """forward_tts.py:848-862 without the host-side managers (tokenizer / AudioProcessor are built by the caller)."""
        return ForwardTTS(copy.deepcopy(config))

    # ------------------------------------------------------------------ packing
    def _create(self, device):
        a = self.args
        enc, dec = self.encoder.encoder.fft_layers, self.decoder.decoder.transformer_block.fft_layers
        ep, dp = a.encoder_params, a.decoder_params
        proj_in = self.proj_g.in_features if hasattr(self, "proj_g") else 0
        pe_len = self.pos_encoder.pe.shape[2] if hasattr(self, "pos_encoder") else 0
        cfg = _lib.ForwardTTSConfigC(
            a.num_chars, a.hidden_channels, a.out_channels, ep["num_heads"], len(enc), ep["hidden_channels_ffn"],
            dp["num_heads"], len(dec), dp["hidden_channels_ffn"], proj_in, a.duration_predictor_hidden_channels,
            a.duration_predictor_kernel_size, int(a.use_pitch), a.pitch_predictor_hidden_channels,
            a.pitch_predictor_kernel_size, a.pitch_embedding_kernel_size, int(a.use_energy),
            a.energy_predictor_hidden_channels, a.energy_predictor_kernel_size, a.energy_embedding_kernel_size, pe_len)
        t = [_host(self.emb.weight)]
        for layer in enc:
            t += layer.weights()
        if proj_in:
            t += _wb(self.proj_g)
        t += self.duration_predictor.ordered_weights()
        if a.use_pitch:
            t += self.pitch_predictor.ordered_weights() + _wb(self.pitch_emb)
        if a.use_energy:
            t += self.energy_predictor.ordered_weights() + _wb(self.energy_emb)
        if pe_len:
            t += [_host(self.pos_encoder.pe[0])]
        for layer in dec:
            t += layer.weights()
        t += _wb(self.decoder.decoder.postnet)
        return self._make("b200tts_forward_tts_create", cfg, t)

    # ------------------------------------------------------------------ conditioning (forward_tts.py:566-577)
    def _set_speaker_input(self, aux_input):
        d_vectors = None if aux_input is None else aux_input.get("d_vectors", None)
        speaker_ids = None if aux_input is None else aux_input.get("speaker_ids", None)
        if d_vectors is not None and speaker_ids is not None:
            raise ValueError("[!] Cannot use d-vectors and speaker-ids together.")
        if speaker_ids is not None and not hasattr(self, "emb_g"):
            raise ValueError("[!] Cannot use speaker-ids without enabling speaker embedding.")
        return speaker_ids if speaker_ids is not None else d_vectors

    def _speaker_vector(self, aux_input, b, device):
        """The [B, C] vector added to the encoder output (emb_g row or d-vector), or the [B, d_vector_dim] d-vector that
        the library projects with proj_g; None without one."""
        g = self._set_speaker_input(aux_input)
        if g is None:
            return None
        g = g.to(device)
        if hasattr(self, "emb_g"):
            g = self.emb_g.weight[g.to(torch.int64).reshape(-1)]
        g = g.to(torch.float32).reshape(g.shape[0], -1).contiguous()
        want = self.proj_g.in_features if hasattr(self, "proj_g") else self.args.hidden_channels
        if g.shape != (b, want):
            raise ValueError(f"tts_b200.ForwardTTS: speaker vector of shape {tuple(g.shape)}, the model takes "
                             f"[{b}, {want}]")
        return g

    # ------------------------------------------------------------------ inference (forward_tts.py:672-714)
    @torch.no_grad()
    def inference(self, x, aux_input={"d_vectors": None, "speaker_ids": None}):  # pylint: disable=dangerous-default-value
        """x int64 [B, T] (CUDA) -> dict(model_outputs [B, T_de, C_out], alignments [B, T_de, T], pitch / energy
        [B, 1, T] or None, durations_log [B, 1, T]) plus durations [B, T] (frames per token) and y_lengths (int64 [B]).

        ``aux_input["x_lengths"]`` (optional) gives each row's token count; the rows past it are padding.  Outputs are
        zero past each row's end.  One host read, of the longest utterance's frame count, sizes the decoder."""
        self._set_speaker_input(aux_input)
        _lib.require_cuda(x, "x")
        dev = x.device
        tok = x.to(torch.int64).contiguous()
        b, tt = tok.shape
        x_lengths = aux_input.get("x_lengths", None) if aux_input is not None else None
        if x_lengths is None:
            x_lengths = torch.full((b,), tt, dtype=torch.int64, device=dev)
        lens = x_lengths.to(device=dev, dtype=torch.int64).contiguous()
        if lens.shape != (b,):
            raise ValueError(f"tts_b200.ForwardTTS: x_lengths must be [{b}], got {tuple(lens.shape)}")
        if tt == 1 or bool((lens == 1).any()):
            # the reference's o_en.squeeze() (:691) also drops the time axis of a one-token utterance
            raise RuntimeError("tts_b200.ForwardTTS: a one-token input fails in the reference's duration predictor "
                               "(o_en.squeeze() drops its time axis)")
        g = self._speaker_vector(aux_input, b, dev)
        a = self.args
        f32 = dict(dtype=torch.float32, device=dev)
        o_en = torch.empty((b, a.hidden_channels, tt), **f32)
        logw = torch.empty((b, 1, tt), **f32)
        pitch = torch.empty((b, 1, tt), **f32) if a.use_pitch else None
        energy = torch.empty((b, 1, tt), **f32) if a.use_energy else None
        x_mask = torch.empty((b, 1, tt), **f32)
        dur = torch.empty((b, tt), **f32)
        cum = torch.empty((b, tt), **f32)
        y_lengths = torch.empty((b,), dtype=torch.int64, device=dev)
        meta = torch.empty((2,), dtype=torch.int64, device=dev)
        h = self.handle(dev)
        L = _lib.lib()
        st = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            ws = _lib.workspace(dev, L.b200tts_forward_tts_encode_workspace_bytes(h, b, tt), "forward_tts")
            rc = L.b200tts_forward_tts_encode(h, _lib.ptr(tok), _lib.ptr(lens), _lib.ptr(g),
                                              ctypes.c_float(float(self.length_scale)), b, tt, _lib.ptr(o_en),
                                              _lib.ptr(logw), _lib.ptr(pitch), _lib.ptr(energy), _lib.ptr(x_mask),
                                              _lib.ptr(dur), _lib.ptr(cum), _lib.ptr(y_lengths), _lib.ptr(meta),
                                              _lib.ptr(ws), ctypes.c_size_t(ws.numel()), st)
            _lib.check(rc, "forward_tts_encode")
            t_dec = int(meta[0].item())     # the one host read: y_max_length of sequence_mask(y_lengths, None)
            if hasattr(self, "pos_encoder") and t_dec > self.pos_encoder.pe.size(2):
                raise RuntimeError(f"Sequence is {t_dec} but PositionalEncoding is limited to "
                                   f"{self.pos_encoder.pe.size(2)}. See max_len argument.")
            attn = torch.empty((b, t_dec, tt), **f32)
            mel = torch.empty((b, t_dec, a.out_channels), **f32)
            ws = _lib.workspace(dev, L.b200tts_forward_tts_decode_workspace_bytes(h, b, t_dec), "forward_tts")
            rc = L.b200tts_forward_tts_decode(h, _lib.ptr(o_en), _lib.ptr(x_mask), _lib.ptr(cum), _lib.ptr(y_lengths),
                                              b, tt, t_dec, _lib.ptr(attn), _lib.ptr(mel), _lib.ptr(ws),
                                              ctypes.c_size_t(ws.numel()), st)
            _lib.check(rc, "forward_tts_decode")
        return {"model_outputs": mel, "alignments": attn, "pitch": pitch, "energy": energy, "durations_log": logw,
                "durations": dur, "y_lengths": y_lengths}

    # ------------------------------------------------------------------ out of scope
    def forward(self, *args, **kwargs):
        raise NotImplementedError("tts_b200.ForwardTTS implements inference only; training (forward) is out of scope")

    # ------------------------------------------------------------------ checkpoints (forward_tts.py:830-837)
    def load_checkpoint(self, config, checkpoint_path, eval=False, cache=False):  # pylint: disable=unused-argument, redefined-builtin
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        self._drop_handle()
        if eval:
            self.eval()
            assert not self.training


def attention(qkv, lengths, num_heads, out=None):
    """Self-attention of the decoder kernel over a fused [B, 3C, T] q|k|v CUDA tensor (rows q | k | v, heads of
    C / num_heads channels), per row over its first ``lengths[b]`` frames: softmax((q d^-1/2) k^T) v -> [B, C, T],
    zero past each row's length.  Heads need d % 8 == 0 and d <= 384."""
    _lib.require_cuda(qkv, "qkv")
    qkv = qkv.to(torch.float32).contiguous()
    b, c3, t = qkv.shape
    c = c3 // 3
    lens = lengths.to(device=qkv.device, dtype=torch.int32).contiguous()
    out = torch.empty((b, c, t), dtype=torch.float32, device=qkv.device) if out is None else out
    with torch.cuda.device(qkv.device):
        rc = _lib.lib().b200tts_attention_tc3(_lib.ptr(qkv), _lib.ptr(lens), b, c, num_heads, t, t, _lib.ptr(out),
                                              _lib.stream_ptr(qkv.device))
    _lib.check(rc, "attention_tc3")
    return out
