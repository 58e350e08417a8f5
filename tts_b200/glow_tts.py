"""Drop-in for the inference path of TTS.tts.models.glow_tts.GlowTTS (TTS/tts/models/glow_tts.py:22-557) and the
model-side fields of its config (TTS/tts/configs/glow_tts_config.py:101-171), on sm_90a kernels.

The whole of ``GlowTTS.inference`` runs in one library handle: text encoder, duration predictor, durations / path /
expanded prior and the Glow decoder in reverse.  Its ``[B, T', C]`` mel output feeds ``tts_b200.vocoder.vocoder_input``
and a HiFiGAN ``GAN`` / ``setup_generator`` vocoder directly.

Kept surface: ``GlowTTS(config, ap, tokenizer, speaker_manager)``, ``GlowTTS.init_from_config``,
``GlowTTS.inference(x, aux_input, *, noise=None)`` -> the reference's 7-key dict (plus ``durations`` and
``y_lengths``), ``load_checkpoint(config, path, eval)``, ``store_inverse`` and the reference ``state_dict`` keys.
Built for ``encoder_type="rel_pos_transformer"`` (the only encoder the released models use); training, MAS and the
data-dependent initialisation raise ``NotImplementedError``.
"""
import ctypes
from dataclasses import asdict, dataclass, field

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.utils import parametrize

from . import _lib
from .layers import WN, DurationPredictor, EngineModule, _Attention, _FFN, _host, _LayerNorm1, _wb


def _cfg(config, key, default=None):
    if isinstance(config, dict):
        return config.get(key, default)
    return getattr(config, key, default)


@dataclass
class GlowTTSConfig:
    """The model-side fields of TTS/tts/configs/glow_tts_config.py with the reference defaults.  The reference
    declares ``encoder_params`` and ``inference_noise_scale`` twice; a dataclass keeps the later declaration, so the
    defaults are ``inference_noise_scale = 0.0`` and ``encoder_params`` with ``input_length: None``."""
    model: str = "glow_tts"
    num_chars: int = None
    encoder_type: str = "rel_pos_transformer"
    encoder_params: dict = field(default_factory=lambda: {"kernel_size": 3, "dropout_p": 0.1, "num_layers": 6,
                                                          "num_heads": 2, "hidden_channels_ffn": 768,
                                                          "input_length": None})
    use_encoder_prenet: bool = True
    hidden_channels_enc: int = 192
    hidden_channels_dec: int = 192
    hidden_channels_dp: int = 256
    dropout_p_dp: float = 0.1
    dropout_p_dec: float = 0.05
    mean_only: bool = True
    out_channels: int = 80
    num_flow_blocks_dec: int = 12
    inference_noise_scale: float = 0.0
    kernel_size_dec: int = 5
    dilation_rate: int = 1
    num_block_layers: int = 4
    num_speakers: int = 0
    c_in_channels: int = 0
    num_splits: int = 4
    num_squeeze: int = 2
    sigmoid_scale: bool = False
    d_vector_dim: int = 0
    data_dep_init_steps: int = 10
    style_wav_for_test: str = None
    length_scale: float = 1.0
    use_speaker_embedding: bool = False
    speakers_file: str = None
    use_d_vector_file: bool = False
    d_vector_file: str = False

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


# ----------------------------------------------------------------------------- parameter containers
class _ResidualConv1dLayerNormBlock(nn.Module):
    """Parameters of TTS/tts/layers/glow_tts/glow.py:11-53 (the encoder prenet)."""

    def __init__(self, in_channels, hidden_channels, out_channels, kernel_size, num_layers):
        super().__init__()
        self.conv_layers = nn.ModuleList()
        self.norm_layers = nn.ModuleList()
        for i in range(num_layers):
            self.conv_layers.append(nn.Conv1d(in_channels if i == 0 else hidden_channels, hidden_channels, kernel_size,
                                              padding=kernel_size // 2))
            self.norm_layers.append(_LayerNorm1(hidden_channels))
        self.proj = nn.Conv1d(hidden_channels, out_channels, 1)
        self.proj.weight.data.zero_()
        self.proj.bias.data.zero_()


class _Transformer(nn.Module):
    """Parameters of RelativePositionTransformer (glow_tts/transformer.py:343-409) as Glow-TTS builds it: no relative
    window, layer_norm_type "1", in = hidden = out channels."""

    def __init__(self, hidden_channels, hidden_channels_ffn, num_heads, num_layers, kernel_size=1, dropout_p=0.0,
                 input_length=None, rel_attn_window_size=None, layer_norm_type="1"):
        super().__init__()
        if rel_attn_window_size is not None or layer_norm_type != "1" or input_length is not None:
            raise NotImplementedError("tts_b200.GlowTTS: the encoder is built without a relative window, with "
                                      "layer_norm_type '1' and input_length None (GlowTTSConfig's encoder)")
        self.attn_layers = nn.ModuleList()
        self.norm_layers_1 = nn.ModuleList()
        self.ffn_layers = nn.ModuleList()
        self.norm_layers_2 = nn.ModuleList()
        for _ in range(num_layers):
            self.attn_layers.append(_Attention(hidden_channels, hidden_channels, num_heads))
            self.norm_layers_1.append(_LayerNorm1(hidden_channels))
            self.ffn_layers.append(_FFN(hidden_channels, hidden_channels, hidden_channels_ffn, kernel_size))
            self.norm_layers_2.append(_LayerNorm1(hidden_channels))


class _Encoder(nn.Module):
    """Parameters of TTS/tts/layers/glow_tts/encoder.py:78-141 for encoder_type "rel_pos_transformer"."""

    def __init__(self, num_chars, out_channels, hidden_channels, hidden_channels_dp, encoder_type, encoder_params,
                 dropout_p_dp=0.1, mean_only=False, use_prenet=True, c_in_channels=0):
        super().__init__()
        if encoder_type.lower() != "rel_pos_transformer":
            raise NotImplementedError(f"tts_b200.GlowTTS: encoder_type {encoder_type!r} is not built "
                                      "(rel_pos_transformer only)")
        self.hidden_channels, self.out_channels = hidden_channels, out_channels
        self.mean_only, self.use_prenet, self.c_in_channels = mean_only, use_prenet, c_in_channels
        self.emb = nn.Embedding(num_chars, hidden_channels)
        nn.init.normal_(self.emb.weight, 0.0, hidden_channels ** -0.5)
        if use_prenet:
            self.prenet = _ResidualConv1dLayerNormBlock(hidden_channels, hidden_channels, hidden_channels, 5, 3)
        p = dict(encoder_params)
        p.pop("dropout_p", None)
        self.encoder = _Transformer(hidden_channels, p.pop("hidden_channels_ffn"), p.pop("num_heads"),
                                    p.pop("num_layers"), **p)
        self.proj_m = nn.Conv1d(hidden_channels, out_channels, 1)
        if not mean_only:
            self.proj_s = nn.Conv1d(hidden_channels, out_channels, 1)
        self.duration_predictor = DurationPredictor(hidden_channels + c_in_channels, hidden_channels_dp, 3, dropout_p_dp)


class _ActNorm(nn.Module):
    """Parameters of TTS/tts/layers/generic/normalization.py:66-86."""

    def __init__(self, channels):
        super().__init__()
        self.logs = nn.Parameter(torch.zeros(1, channels, 1))
        self.bias = nn.Parameter(torch.zeros(1, channels, 1))


class _InvConvNear(nn.Module):
    """Parameters of TTS/tts/layers/glow_tts/glow.py:70-100 (+ ``weight_inv`` after ``store_inverse``, :139-141)."""

    def __init__(self, channels, num_splits=4):
        super().__init__()
        assert num_splits % 2 == 0
        self.num_splits = num_splits
        self.weight_inv = None
        w_init = torch.linalg.qr(torch.FloatTensor(num_splits, num_splits).normal_(), "complete")[0]
        if torch.det(w_init) < 0:
            w_init[:, 0] = -1 * w_init[:, 0]
        self.weight = nn.Parameter(w_init)

    def inverse(self):
        """The matrix the reverse pass multiplies by (glow.py:119-123), computed on the host."""
        if self.weight_inv is not None:
            return _host(self.weight_inv)
        return torch.inverse(_host(self.weight).float())

    def store_inverse(self):
        self.weight_inv = nn.Parameter(torch.inverse(self.weight.detach().float()).to(self.weight.dtype),
                                       requires_grad=False)


class _CouplingBlock(nn.Module):
    """Parameters of TTS/tts/layers/glow_tts/glow.py:167-199."""

    def __init__(self, in_channels, hidden_channels, kernel_size, dilation_rate, num_layers, c_in_channels=0,
                 dropout_p=0):
        super().__init__()
        self.start = torch.nn.utils.parametrizations.weight_norm(torch.nn.Conv1d(in_channels // 2, hidden_channels, 1))
        self.end = torch.nn.Conv1d(hidden_channels, in_channels, 1)
        self.end.weight.data.zero_()
        self.end.bias.data.zero_()
        self.wn = WN(hidden_channels, hidden_channels, kernel_size, dilation_rate, num_layers, c_in_channels, dropout_p)

    def store_inverse(self):   # WN.remove_weight_norm, wavenet.py:117-123
        for m in ([self.wn.cond_layer] if self.wn.c_in_channels else []) + list(self.wn.in_layers) + \
                list(self.wn.res_skip_layers):
            parametrize.remove_parametrizations(m, "weight")


class _Decoder(nn.Module):
    """Parameters of TTS/tts/layers/glow_tts/decoder.py:68-111: per block ActNorm, InvConvNear, CouplingBlock."""

    def __init__(self, in_channels, hidden_channels, kernel_size, dilation_rate, num_flow_blocks, num_coupling_layers,
                 dropout_p=0.0, num_splits=4, num_squeeze=2, c_in_channels=0):
        super().__init__()
        c = in_channels * num_squeeze
        self.flows = nn.ModuleList()
        for _ in range(num_flow_blocks):
            self.flows.append(_ActNorm(c))
            self.flows.append(_InvConvNear(c, num_splits))
            self.flows.append(_CouplingBlock(c, hidden_channels, kernel_size, dilation_rate, num_coupling_layers,
                                             c_in_channels, dropout_p))


# ----------------------------------------------------------------------------- model
class GlowTTS(EngineModule):
    """Glow-TTS text -> mel synthesiser, inference path on sm_90a kernels."""

    _destroy = "b200tts_glow_tts_destroy"

    def __init__(self, config, ap=None, tokenizer=None, speaker_manager=None):
        super().__init__()
        self.config, self.ap, self.tokenizer, self.speaker_manager = config, ap, tokenizer, speaker_manager
        for key in ("num_chars", "encoder_type", "encoder_params", "use_encoder_prenet", "hidden_channels_enc",
                    "hidden_channels_dec", "hidden_channels_dp", "dropout_p_dp", "dropout_p_dec", "mean_only",
                    "out_channels", "num_flow_blocks_dec", "inference_noise_scale", "kernel_size_dec", "dilation_rate",
                    "num_block_layers", "num_speakers", "num_splits", "num_squeeze", "sigmoid_scale",
                    "length_scale", "data_dep_init_steps"):
            setattr(self, key, _cfg(config, key))
        if tokenizer is not None:   # BaseTTS._set_model_args (base_tts.py:61-66)
            self.num_chars = tokenizer.characters.num_chars
        self.decoder_output_dim = self.out_channels
        self.init_multispeaker(config)
        self.encoder = _Encoder(self.num_chars, self.out_channels, self.hidden_channels_enc, self.hidden_channels_dp,
                                self.encoder_type, self.encoder_params, self.dropout_p_dp, self.mean_only,
                                self.use_encoder_prenet, self.c_in_channels)
        self.decoder = _Decoder(self.out_channels, self.hidden_channels_dec, self.kernel_size_dec, self.dilation_rate,
                                self.num_flow_blocks_dec, self.num_block_layers, self.dropout_p_dec, self.num_splits,
                                self.num_squeeze, self.c_in_channels)

    def init_multispeaker(self, config):
        """glow_tts.py:107-135."""
        self.embedded_speaker_dim = 0
        if self.speaker_manager is not None:
            self.num_speakers = self.speaker_manager.num_speakers
        if _cfg(config, "use_d_vector_file", False):
            dim = _cfg(config, "d_vector_dim", None)
            self.embedded_speaker_dim = dim if dim is not None else 512
            if self.speaker_manager is not None:
                assert dim == self.speaker_manager.embedding_dim, \
                    " [!] d-vector dimension mismatch b/w config and speaker manager."
        if _cfg(config, "use_speaker_embedding", False) and not _cfg(config, "use_d_vector_file", False):
            self.embedded_speaker_dim = self.hidden_channels_enc
            self.emb_g = nn.Embedding(self.num_speakers, self.hidden_channels_enc)
            nn.init.uniform_(self.emb_g.weight, -0.1, 0.1)
        self.c_in_channels = self.embedded_speaker_dim

    @staticmethod
    def init_from_config(config, samples=None, verbose=True):  # pylint: disable=unused-argument
        """glow_tts.py:542-557 without the host-side managers (tokenizer / AudioProcessor are built by the caller)."""
        return GlowTTS(config)

    # ------------------------------------------------------------------ packing
    def _create(self, device):
        e, n_dec = self.encoder, self.num_flow_blocks_dec
        p = self.encoder_params
        cfg = _lib.GlowTTSConfigC(self.num_chars, self.out_channels, self.hidden_channels_enc, p["hidden_channels_ffn"],
                                  p["num_heads"], p["num_layers"], p.get("kernel_size", 1), int(self.use_encoder_prenet),
                                  int(self.mean_only), self.hidden_channels_dp, self.c_in_channels,
                                  self.hidden_channels_dec, self.kernel_size_dec, self.dilation_rate, n_dec,
                                  self.num_block_layers, self.num_splits, self.num_squeeze, int(self.sigmoid_scale))
        ln = lambda n: [_host(n.gamma.reshape(-1)), _host(n.beta.reshape(-1))]   # noqa: E731
        t = [_host(e.emb.weight)]
        if self.use_encoder_prenet:
            for conv, norm in zip(e.prenet.conv_layers, e.prenet.norm_layers):
                t += _wb(conv) + ln(norm)
            t += _wb(e.prenet.proj)
        enc = e.encoder
        for a, n1, f, n2 in zip(enc.attn_layers, enc.norm_layers_1, enc.ffn_layers, enc.norm_layers_2):
            t += _wb(a.conv_q) + _wb(a.conv_k) + _wb(a.conv_v) + _wb(a.conv_o) + ln(n1) + _wb(f.conv_1) + _wb(f.conv_2)
            t += ln(n2)
        t += _wb(e.proj_m) + ([] if self.mean_only else _wb(e.proj_s))
        dp = e.duration_predictor
        t += _wb(dp.conv_1) + ln(dp.norm_1) + _wb(dp.conv_2) + ln(dp.norm_2) + _wb(dp.proj)
        fl = self.decoder.flows
        for n in range(n_dec):
            an, ic, cb = fl[3 * n], fl[3 * n + 1], fl[3 * n + 2]
            t += [_host(an.logs.reshape(-1)), _host(an.bias.reshape(-1)), ic.inverse().contiguous()]
            t += _wb(cb.start) + cb.wn.ordered_weights() + _wb(cb.end)
        return self._make("b200tts_glow_tts_create", cfg, t)

    # ------------------------------------------------------------------ conditioning (glow_tts.py:162-191)
    def _set_speaker_input(self, aux_input):
        d_vectors = None if aux_input is None else aux_input.get("d_vectors", None)
        speaker_ids = None if aux_input is None else aux_input.get("speaker_ids", None)
        if d_vectors is not None and speaker_ids is not None:
            raise ValueError("[!] Cannot use d-vectors and speaker-ids together.")
        if speaker_ids is not None and not hasattr(self, "emb_g"):
            raise ValueError("[!] Cannot use speaker-ids without enabling speaker embedding.")
        return speaker_ids if speaker_ids is not None else d_vectors

    def _speaker_embedding(self, aux_input, device):
        """The l2-normalised speaker vector [B, c_in] (the reference's [B, c_in, 1] without the last axis)."""
        g = self._set_speaker_input(aux_input)
        if g is None:
            return None
        g = g.to(device)
        if hasattr(self, "emb_g"):
            if not g.size():
                g = g.unsqueeze(0)
            return F.normalize(self.emb_g(g)).to(torch.float32).contiguous()
        return F.normalize(g).to(torch.float32).contiguous()

    # ------------------------------------------------------------------ inference (glow_tts.py:341-374)
    @torch.no_grad()
    def inference(self, x, aux_input={"x_lengths": None, "d_vectors": None, "speaker_ids": None}, *,
                  noise=None):  # pylint: disable=dangerous-default-value
        """x int64 [B, T] (CUDA) -> dict(model_outputs [B, T', C], logdet None, y_mean, y_log_scale [B, T_dec, C],
        alignments [B, T_dec, T], durations_log, total_durations_log [B, T, 1]), plus durations (w_ceil [B, 1, T]) and
        y_lengths (int64 [B]).  As in the reference, the [B, T, C] outputs are transposed views.

        ``noise`` [B, C, T_dec] replaces the ``torch.randn_like(y_mean)`` draw (:361) so that runs are reproducible;
        with ``inference_noise_scale == 0`` nothing is drawn (the draw is multiplied by zero).  One host read, of the
        longest utterance's frame count, sizes the decoder."""
        self._set_speaker_input(aux_input)
        _lib.require_cuda(x, "x")
        dev = x.device
        tok = x.to(torch.int64).contiguous()
        b, tt = tok.shape
        x_lengths = aux_input.get("x_lengths", None) if aux_input is not None else None
        if x_lengths is None:
            x_lengths = torch.full((b,), tt, dtype=torch.int64, device=dev)
        lens = x_lengths.to(device=dev, dtype=torch.int64).contiguous()
        g = self._speaker_embedding(aux_input, dev)
        if self.c_in_channels > 0 and g is None:
            raise ValueError("tts_b200.GlowTTS: multi-speaker model needs speaker_ids or d_vectors")
        if g is not None and (self.c_in_channels == 0 or g.shape != (b, self.c_in_channels)):
            raise ValueError(f"tts_b200.GlowTTS: speaker vector of shape {tuple(g.shape)}, the model takes "
                             f"[{b}, {self.c_in_channels}]")
        c = self.out_channels
        f32 = dict(dtype=torch.float32, device=dev)
        o_stats = torch.empty((b, 2 * c, tt), **f32)
        logw = torch.empty((b, 1, tt), **f32)
        x_mask = torch.empty((b, 1, tt), **f32)
        w_ceil = torch.empty((b, 1, tt), **f32)
        cum = torch.empty((b, tt), **f32)
        dur_log = torch.empty((b, 1, tt), **f32)
        y_lengths = torch.empty((b,), dtype=torch.int64, device=dev)
        meta = torch.empty((2,), dtype=torch.int64, device=dev)
        h = self.handle(dev)
        L = _lib.lib()
        st = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            ws = _lib.workspace(dev, L.b200tts_glow_tts_workspace_bytes(h, b, tt, 0), "glow_tts")
            rc = L.b200tts_glow_tts_encode(h, _lib.ptr(tok), _lib.ptr(lens), _lib.ptr(g),
                                           ctypes.c_float(float(self.length_scale)), b, tt, _lib.ptr(o_stats),
                                           _lib.ptr(logw), _lib.ptr(x_mask), _lib.ptr(w_ceil), _lib.ptr(cum),
                                           _lib.ptr(dur_log), _lib.ptr(y_lengths), _lib.ptr(meta), _lib.ptr(ws),
                                           ctypes.c_size_t(ws.numel()), st)
            _lib.check(rc, "glow_tts_encode")
            t_dec = int(meta[0].item())     # the one host read: y_max_length of sequence_mask(y_lengths, None)
            scale = float(self.inference_noise_scale)
            nz = None
            if scale != 0.0:
                nz = torch.randn((b, c, t_dec), **f32) if noise is None else noise.to(**f32).contiguous()
                if nz.shape != (b, c, t_dec):
                    raise ValueError(f"tts_b200.GlowTTS: noise must be [{b}, {c}, {t_dec}], got {tuple(nz.shape)}")
            attn = torch.empty((b, tt, t_dec), **f32)
            y_mean = torch.empty((b, c, t_dec), **f32)
            y_log_scale = torch.empty((b, c, t_dec), **f32)
            mel = torch.empty((b, c, (t_dec // self.num_squeeze) * self.num_squeeze), **f32)
            ws = _lib.workspace(dev, L.b200tts_glow_tts_workspace_bytes(h, b, tt, t_dec), "glow_tts")
            rc = L.b200tts_glow_tts_decode(h, _lib.ptr(o_stats), _lib.ptr(x_mask), _lib.ptr(cum), _lib.ptr(y_lengths),
                                           _lib.ptr(g), _lib.ptr(nz), ctypes.c_float(scale), b, tt, t_dec,
                                           _lib.ptr(attn), _lib.ptr(y_mean), _lib.ptr(y_log_scale), _lib.ptr(mel),
                                           _lib.ptr(ws), ctypes.c_size_t(ws.numel()), st)
            _lib.check(rc, "glow_tts_decode")
        return {"model_outputs": mel.transpose(1, 2), "logdet": None, "y_mean": y_mean.transpose(1, 2),
                "y_log_scale": y_log_scale.transpose(1, 2), "alignments": attn.transpose(1, 2),
                "durations_log": logw.transpose(1, 2), "total_durations_log": dur_log.transpose(1, 2),
                "durations": w_ceil, "y_lengths": y_lengths}

    # ------------------------------------------------------------------ out of scope
    def forward(self, *args, **kwargs):
        raise NotImplementedError("tts_b200.GlowTTS implements inference only; training (forward) is out of scope")

    def inference_with_MAS(self, *args, **kwargs):  # pylint: disable=invalid-name
        raise NotImplementedError("tts_b200.GlowTTS: inference_with_MAS (teacher-forced analysis) is out of scope")

    def decoder_inference(self, *args, **kwargs):
        raise NotImplementedError("tts_b200.GlowTTS: decoder_inference (decoder round trip) is out of scope")

    def unlock_act_norm_layers(self):
        raise NotImplementedError("tts_b200.GlowTTS: data-dependent ActNorm initialisation is training only")

    # ------------------------------------------------------------------ checkpoints (glow_tts.py:519-530)
    def store_inverse(self):
        for f in self.decoder.flows:
            if isinstance(f, (_InvConvNear, _CouplingBlock)):
                f.store_inverse()
        self._drop_handle()

    def load_checkpoint(self, config, checkpoint_path, eval=False):  # pylint: disable=unused-argument, redefined-builtin
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        self._drop_handle()
        if eval:
            self.eval()
            self.store_inverse()
            assert not self.training
