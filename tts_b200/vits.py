"""Drop-in for the inference path of TTS.tts.models.vits.Vits
(/root/reference/TTS/tts/models/vits.py:603-1173) plus the config dataclasses it reads
(VitsArgs :365-600, VitsAudioConfig :216-224, VitsConfig TTS/tts/configs/vits_config.py:8-176).

``coqpit`` is not required: the dataclasses below carry the same field names and defaults and accept
either attribute or item access, so a real ``VitsConfig`` (coqpit) object works as well.
Kept surface: ``Vits(config, ap, tokenizer, speaker_manager, language_manager)``,
``Vits.init_from_config``, ``Vits.inference(x, aux_input)`` -> the same 8-key dict,
``Vits.load_checkpoint``, and the reference ``state_dict`` key names.
"""
from dataclasses import asdict, dataclass, field
from typing import Dict, List

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .hifigan import HifiganGenerator
from .layers import upsample_linear
from .layers import (DurationPredictor, EngineModule, PosteriorEncoder, ResidualCouplingBlocks, StochasticDurationPredictor,
                     TextEncoder, durations_to_path, expand_prior)


class _ItemAccess:
    def __getitem__(self, k):
        return getattr(self, k)

    def __setitem__(self, k, v):
        setattr(self, k, v)

    def __contains__(self, k):
        return hasattr(self, k)

    def items(self):
        return asdict(self).items()

    def get(self, k, default=None):
        return getattr(self, k, default)


@dataclass
class VitsAudioConfig(_ItemAccess):
    fft_size: int = 1024
    sample_rate: int = 22050
    win_length: int = 1024
    hop_length: int = 256
    num_mels: int = 80
    mel_fmin: int = 0
    mel_fmax: int = None


@dataclass
class VitsArgs(_ItemAccess):
    num_chars: int = 100
    out_channels: int = 513
    spec_segment_size: int = 32
    hidden_channels: int = 192
    hidden_channels_ffn_text_encoder: int = 768
    num_heads_text_encoder: int = 2
    num_layers_text_encoder: int = 6
    kernel_size_text_encoder: int = 3
    dropout_p_text_encoder: float = 0.1
    dropout_p_duration_predictor: float = 0.5
    kernel_size_posterior_encoder: int = 5
    dilation_rate_posterior_encoder: int = 1
    num_layers_posterior_encoder: int = 16
    kernel_size_flow: int = 5
    dilation_rate_flow: int = 1
    num_layers_flow: int = 4
    resblock_type_decoder: str = "1"
    resblock_kernel_sizes_decoder: List[int] = field(default_factory=lambda: [3, 7, 11])
    resblock_dilation_sizes_decoder: List[List[int]] = field(default_factory=lambda: [[1, 3, 5], [1, 3, 5], [1, 3, 5]])
    upsample_rates_decoder: List[int] = field(default_factory=lambda: [8, 8, 2, 2])
    upsample_initial_channel_decoder: int = 512
    upsample_kernel_sizes_decoder: List[int] = field(default_factory=lambda: [16, 16, 4, 4])
    periods_multi_period_discriminator: List[int] = field(default_factory=lambda: [2, 3, 5, 7, 11])
    use_sdp: bool = True
    noise_scale: float = 1.0
    inference_noise_scale: float = 0.667
    length_scale: float = 1
    noise_scale_dp: float = 1.0
    inference_noise_scale_dp: float = 1.0
    max_inference_len: int = None
    init_discriminator: bool = True
    use_spectral_norm_disriminator: bool = False
    use_speaker_embedding: bool = False
    num_speakers: int = 0
    speakers_file: str = None
    d_vector_file: List[str] = None
    speaker_embedding_channels: int = 256
    use_d_vector_file: bool = False
    d_vector_dim: int = 0
    detach_dp_input: bool = True
    use_language_embedding: bool = False
    embedded_language_dim: int = 4
    num_languages: int = 0
    language_ids_file: str = None
    use_speaker_encoder_as_loss: bool = False
    speaker_encoder_config_path: str = ""
    speaker_encoder_model_path: str = ""
    condition_dp_on_speaker: bool = True
    freeze_encoder: bool = False
    freeze_DP: bool = False
    freeze_PE: bool = False
    freeze_flow_decoder: bool = False
    freeze_waveform_decoder: bool = False
    encoder_sample_rate: int = None
    interpolate_z: bool = True
    reinit_DP: bool = False
    reinit_text_encoder: bool = False


@dataclass
class VitsConfig(_ItemAccess):
    """The fields of TTS/tts/configs/vits_config.py:8-176 the inference path reads."""
    model: str = "vits"
    model_args: VitsArgs = field(default_factory=VitsArgs)
    audio: VitsAudioConfig = field(default_factory=VitsAudioConfig)
    add_blank: bool = True
    num_speakers: int = 0
    use_speaker_embedding: bool = False
    speakers_file: str = None
    speaker_embedding_channels: int = 256
    language_ids_file: str = None
    use_language_embedding: bool = False
    use_d_vector_file: bool = False
    d_vector_file: List[str] = None
    d_vector_dim: int = None

    def __post_init__(self):  # vits_config.py:173-176: mirror model_args onto the top level
        for key, val in self.model_args.items():
            if hasattr(self, key) and key not in ("model_args", "audio"):
                setattr(self, key, val)


class _Stage:
    """Optional CUDA-event bracket around one stage of Vits.inference (bench.py sets model._stage_events)."""

    def __init__(self, model, name):
        self.events, self.name = getattr(model, "_stage_events", None), name

    def __enter__(self):
        if self.events is not None:
            self.start = torch.cuda.Event(enable_timing=True)
            self.start.record()
        return self

    def __exit__(self, *exc):
        if self.events is not None:
            end = torch.cuda.Event(enable_timing=True)
            end.record()
            self.events.append((self.name, self.start, end))
        return False


def _get(obj, key, default=None):
    if isinstance(obj, dict):
        return obj.get(key, default)
    return getattr(obj, key, default)


class Vits(nn.Module):
    """VITS end-to-end synthesiser, inference path on sm_90a kernels."""

    def __init__(self, config, ap=None, tokenizer=None, speaker_manager=None, language_manager=None):
        super().__init__()
        self.config = config
        self.args = _get(config, "model_args", config)
        self.ap, self.tokenizer = ap, tokenizer
        self.speaker_manager, self.language_manager = speaker_manager, language_manager
        a = self.args
        self.init_multispeaker(config)
        self.init_multilingual(config)
        self.length_scale = a.length_scale
        self.noise_scale = a.noise_scale
        self.inference_noise_scale = a.inference_noise_scale
        self.inference_noise_scale_dp = a.inference_noise_scale_dp
        self.noise_scale_dp = a.noise_scale_dp
        self.max_inference_len = a.max_inference_len
        self.spec_segment_size = a.spec_segment_size
        # tts_b200 extension (default off = the reference's batch semantics, padded tail included): skip the padded frames
        # of a batch in the flow and the decoder.  Every sample below ``wav_lengths[b]`` stays bit-identical; the padded
        # tail of ``model_outputs`` (the decoder's response to zero input, which no caller keeps) becomes zero.
        self.trim_padding = False
        if a.encoder_sample_rate:   # vits.py:809-810 (the training-only torchaudio resampler is not needed here)
            self.interpolate_factor = _get(config, "audio")["sample_rate"] / a.encoder_sample_rate

        self.text_encoder = TextEncoder(a.num_chars, a.hidden_channels, a.hidden_channels,
                                        a.hidden_channels_ffn_text_encoder, a.num_heads_text_encoder,
                                        a.num_layers_text_encoder, a.kernel_size_text_encoder,
                                        a.dropout_p_text_encoder, language_emb_dim=self.embedded_language_dim)
        self.posterior_encoder = PosteriorEncoder(a.out_channels, a.hidden_channels, a.hidden_channels,
                                                  kernel_size=a.kernel_size_posterior_encoder,
                                                  dilation_rate=a.dilation_rate_posterior_encoder,
                                                  num_layers=a.num_layers_posterior_encoder,
                                                  cond_channels=self.embedded_speaker_dim)
        self.flow = ResidualCouplingBlocks(a.hidden_channels, a.hidden_channels, kernel_size=a.kernel_size_flow,
                                           dilation_rate=a.dilation_rate_flow, num_layers=a.num_layers_flow,
                                           cond_channels=self.embedded_speaker_dim)
        if a.use_sdp:
            self.duration_predictor = StochasticDurationPredictor(
                a.hidden_channels, 192, 3, a.dropout_p_duration_predictor, 4,
                cond_channels=self.embedded_speaker_dim if a.condition_dp_on_speaker else 0,
                language_emb_dim=self.embedded_language_dim)
        else:  # vits.py:646-654
            self.duration_predictor = DurationPredictor(
                a.hidden_channels, 256, 3, a.dropout_p_duration_predictor,
                cond_channels=self.embedded_speaker_dim, language_emb_dim=self.embedded_language_dim)
        self.waveform_decoder = HifiganGenerator(
            a.hidden_channels, 1, a.resblock_type_decoder, a.resblock_dilation_sizes_decoder,
            a.resblock_kernel_sizes_decoder, a.upsample_kernel_sizes_decoder, a.upsample_initial_channel_decoder,
            a.upsample_rates_decoder, inference_padding=0, cond_channels=self.embedded_speaker_dim,
            conv_pre_weight_norm=False, conv_post_weight_norm=False, conv_post_bias=False)
        # the discriminator (vits.py:719-724) is training-only and intentionally absent

    # ------------------------------------------------------------------ construction helpers (vits.py:730-801)
    @property
    def device(self):
        return next(self.parameters()).device

    def init_multispeaker(self, config):
        self.embedded_speaker_dim = 0
        self.num_speakers = self.args.num_speakers
        if self.speaker_manager:
            self.num_speakers = self.speaker_manager.num_speakers
        if self.args.use_speaker_embedding and self.num_speakers > 0:
            self.embedded_speaker_dim = self.args.speaker_embedding_channels
            self.emb_g = nn.Embedding(self.num_speakers, self.embedded_speaker_dim)
        if self.args.use_d_vector_file:
            if hasattr(self, "emb_g"):
                raise ValueError("[!] Speaker embedding layer already initialized before d_vector settings.")
            self.embedded_speaker_dim = self.args.d_vector_dim

    def init_multilingual(self, config):
        self.embedded_language_dim = 0
        n = self.args.num_languages
        if self.language_manager is not None:
            n = self.language_manager.num_languages
        if self.args.use_language_embedding and n > 0:
            self.num_languages = n
            self.embedded_language_dim = self.args.embedded_language_dim
            self.emb_l = nn.Embedding(self.num_languages, self.embedded_language_dim)
            torch.nn.init.xavier_uniform_(self.emb_l.weight)

    @staticmethod
    def init_from_config(config, samples=None, verbose=True):
        """vits.py:1771-1804 without the host-side managers (tokenizer / AudioProcessor are out of scope)."""
        up = 1
        for u in _get(config, "model_args").upsample_rates_decoder:
            up *= u
        hop = _get(config, "audio").hop_length
        esr = _get(config, "model_args").encoder_sample_rate
        if esr:   # vits.py:1789-1794
            hop = hop * (_get(config, "audio").sample_rate / esr)
        assert up == hop, f" [!] Product of upsample rates must be equal to the hop length - {up} vs {hop}"
        return Vits(config)

    # ------------------------------------------------------------------ conditioning (vits.py:874-905)
    @staticmethod
    def _set_cond_input(aux_input: Dict):
        sid, g, lid, durations = None, None, None, None
        if aux_input.get("speaker_ids", None) is not None:
            sid = aux_input["speaker_ids"]
            if sid.ndim == 0:
                sid = sid.unsqueeze_(0)
        if aux_input.get("d_vectors", None) is not None:
            g = F.normalize(aux_input["d_vectors"]).unsqueeze(-1)
            if g.ndim == 2:
                g = g.unsqueeze_(0)
        if aux_input.get("language_ids", None) is not None:
            lid = aux_input["language_ids"]
            if lid.ndim == 0:
                lid = lid.unsqueeze_(0)
        if aux_input.get("durations", None) is not None:
            durations = aux_input["durations"]
        return sid, g, lid, durations

    @staticmethod
    def _set_x_lengths(x, aux_input):
        if aux_input.get("x_lengths", None) is not None:
            return aux_input["x_lengths"]
        return torch.tensor(x.shape[1:2]).to(x.device)

    # ------------------------------------------------------------------ inference (vits.py:1088-1173)
    @torch.no_grad()
    def inference(self, x, aux_input={"x_lengths": None, "d_vectors": None, "speaker_ids": None,
                                      "language_ids": None, "durations": None}, *, sdp_noise=None,
                  prior_noise=None, return_alignments=True):  # pylint: disable=dangerous-default-value
        """x int64 [B,T_seq] (CUDA) -> dict(model_outputs, alignments, durations, z, z_p, m_p, logs_p, y_mask).

        ``sdp_noise`` [B,2,T_seq] / ``prior_noise`` [B,C,T_dec] (or a callable shape->tensor) replace the two
        random draws of the reference (SURVEY appendix A7) so results can be compared exactly; by default they
        are drawn like the reference does (CPU generator, then device generator)."""
        lat = self._latents(x, aux_input, sdp_noise, prior_noise, return_alignments)
        zin, frame_lengths = lat["zin"], lat["frame_lengths"]
        with _Stage(self, "waveform_decoder"):
            o = self.waveform_decoder(zin, g=lat["g"], lengths=frame_lengths if lat["ragged"] else None)
        hop = o.shape[-1] // max(zin.shape[-1], 1)      # prod(upsample_rates_decoder)
        # the reference's eight keys (vits.py:1163-1172) plus: y_lengths (frames at the text-side rate), logw, and
        # wav_lengths = valid output samples per utterance (after latent upsampling / max_inference_len cropping)
        return {"model_outputs": o, "alignments": lat["attn"], "durations": lat["w_ceil"], "z": lat["z"],
                "z_p": lat["z_p"], "m_p": lat["m_p"], "logs_p": lat["logs_p"], "y_mask": lat["y_mask"],
                "y_lengths": lat["y_lengths"], "logw": lat["logw"], "wav_lengths": frame_lengths * hop}

    @torch.no_grad()
    def inference_stream(self, x, aux_input={"x_lengths": None, "d_vectors": None, "speaker_ids": None,
                                             "language_ids": None, "durations": None}, chunk_frames=32, *,
                         sdp_noise=None, prior_noise=None):  # pylint: disable=dangerous-default-value
        """Streaming ``inference``: a generator of waveform chunks, the first one available long before the whole
        batch is decoded.

        The text encoder, duration predictor, path, flow (and latent upsampling / ``max_inference_len``) run whole, as
        in ``inference``, with its one host read of the decoder length T_dec.  The decoder then runs over consecutive
        windows of ``chunk_frames`` decoder-input frames; each yields ``{"model_outputs": [B, 1, n] waveform chunk,
        "start": index of its first sample, "wav_lengths": [B] valid samples per utterance}``.  Every chunk is
        bit-identical to the same samples of ``inference(...)["model_outputs"]`` with the same noise (no cross-fade:
        each window recomputes its receptive-field halo from the latents), ``trim_padding`` included.  The chunks are
        views of one ``[B, 1, T_dec * hop]`` buffer that later chunks do not overwrite, so earlier ones stay valid.
        Nothing is read back to the host per chunk."""
        if int(chunk_frames) < 1:
            raise ValueError("tts_b200.Vits.inference_stream: chunk_frames must be >= 1")
        lat = self._latents(x, aux_input, sdp_noise, prior_noise, False)
        dec = self.waveform_decoder
        zin = lat["zin"].to(torch.float32).contiguous()
        b, _, t = zin.shape
        hop = dec.hop
        lengths = lat["frame_lengths"].to(torch.int32).contiguous() if lat["ragged"] else None
        wav_lengths = lat["frame_lengths"] * hop
        out = torch.empty((b, 1, t * hop), dtype=torch.float32, device=zin.device)
        for f0 in range(0, t, int(chunk_frames)):
            f1 = min(t, f0 + int(chunk_frames))
            o = dec.forward_window(zin, g=lat["g"], start=f0, end=f1, lengths=lengths, out=out)
            yield {"model_outputs": o, "start": f0 * hop, "wav_lengths": wav_lengths}

    def _latents(self, x, aux_input, sdp_noise, prior_noise, return_alignments):
        """Everything of ``inference`` before the decoder: text encoder -> durations -> path -> flow."""
        _lib.require_cuda(x, "x")
        a = self.args
        sid, g, lid, durations = self._set_cond_input(aux_input)
        if durations is not None:  # vits.py:1141-1143: w = durations.unsqueeze(0), i.e. a single utterance
            assert durations.shape[-1] == x.shape[-1]
            if x.shape[0] != 1:
                raise ValueError("tts_b200.Vits: aux_input['durations'] is defined for batch size 1 (vits.py:1143)")
        x_lengths = self._set_x_lengths(x, aux_input)
        if a.use_speaker_embedding and sid is not None:
            g = self.emb_g(sid.to(x.device)).unsqueeze(-1)
        lang_emb = None
        if a.use_language_embedding and lid is not None:
            lang_emb = self.emb_l(lid.to(x.device)).unsqueeze(-1)
        if self.embedded_speaker_dim > 0 and g is None:
            raise ValueError("tts_b200.Vits: multi-speaker model needs speaker_ids or d_vectors")

        with _Stage(self, "text_encoder"):
            h, stats, x_mask = self.text_encoder.forward_stats(x, x_lengths, lang_emb=lang_emb)
        with _Stage(self, "duration_predictor"):
            logw, meta = None, None
            if durations is not None:
                w = durations.to(device=x.device, dtype=torch.float32).reshape(1, 1, -1)
                w_ceil = torch.ceil(w)
                cum = torch.cumsum(w_ceil.reshape(1, -1), dim=1)
                y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()
            else:
                flag = None
                if a.use_sdp:
                    logw = self.duration_predictor(h, x_mask, g=g if a.condition_dp_on_speaker else None,
                                                   reverse=True, noise_scale=self.inference_noise_scale_dp,
                                                   lang_emb=lang_emb, noise=sdp_noise)
                    # consumed here: a stale flag must not be re-read by a later call that supplies durations
                    flag, self.duration_predictor.last_error_flag = self.duration_predictor.last_error_flag, None
                else:
                    logw = self.duration_predictor(h, x_mask, g=g if a.condition_dp_on_speaker else None,
                                                   lang_emb=lang_emb)
                w_ceil, cum, y_lengths, meta = durations_to_path(logw, x_mask, float(self.length_scale), err_flag=flag)
        # the one host sync of the path: T_dec = max(y_lengths) (sequence_mask(y_lengths, None), helpers.py:53-54),
        # read together with the spline error flag in a single 16-byte D2H copy
        if meta is not None:
            t_dec, bad = (int(v) for v in meta.tolist())
            if bad != 0:
                raise AssertionError("spline discriminant < 0 (TTS/tts/layers/vits/transforms.py:168)")
        else:
            t_dec = int(y_lengths.max().item())
        c = a.hidden_channels
        if prior_noise is None:
            noise = torch.randn((x.shape[0], c, t_dec), dtype=torch.float32, device=x.device)
        elif callable(prior_noise):
            if getattr(prior_noise, "wants_lengths", False):     # per-row draws (parallel.synthesize_batched)
                noise = prior_noise((x.shape[0], c, t_dec), y_lengths.tolist())
            else:
                noise = prior_noise((x.shape[0], c, t_dec))
        else:
            noise = prior_noise
        with _Stage(self, "expand_prior"):
            attn, m_p, logs_p, z_p, y_mask = expand_prior(cum, x_mask, y_lengths, stats, noise,
                                                          float(self.inference_noise_scale), t_dec,
                                                          want_attn=return_alignments)
        frame_lengths = y_lengths            # valid decoder frames per utterance at the decoder's input rate
        ragged = bool(getattr(self, "trim_padding", False)) and x.shape[0] > 1
        with _Stage(self, "flow"):
            z = self.flow(z_p, y_mask, g=g, reverse=True, lengths=y_lengths if ragged else None)
            if a.encoder_sample_rate and a.interpolate_z:   # upsampling_z, vits.py:944-959
                f = self.interpolate_factor
                z = upsample_linear(z, f)
                len_up = y_lengths * f
                y_mask = (torch.arange(float(len_up.max()), device=z.device)[None, :] < len_up[:, None]).to(y_mask.dtype).unsqueeze(1)
                if y_mask.shape[-1] != z.shape[-1]:
                    raise ValueError("tts_b200.Vits: sample_rate / encoder_sample_rate must scale the frame count to an "
                                     "integer (the reference's z * y_mask fails the same way, vits.py:1160)")
                frame_lengths = torch.ceil(len_up).long()    # frames t with t < y_lengths * f, as the rebuilt mask counts
            zin = z * y_mask
            if self.max_inference_len is not None:
                zin = zin[:, :, : self.max_inference_len]
                frame_lengths = torch.clamp_max(frame_lengths, int(self.max_inference_len))
        return {"attn": attn, "w_ceil": w_ceil, "z": z, "z_p": z_p, "m_p": m_p, "logs_p": logs_p, "y_mask": y_mask,
                "y_lengths": y_lengths, "logw": logw, "zin": zin, "frame_lengths": frame_lengths, "ragged": ragged,
                "g": g}

    # ------------------------------------------------------------------ voice conversion (vits.py:1175-1232)
    @torch.no_grad()
    def inference_voice_conversion(self, reference_wav, speaker_id=None, d_vector=None, reference_speaker_id=None,
                                   reference_d_vector=None, *, posterior_noise=None):
        """reference_wav [B,1,T] or [B,T] (CUDA) -> converted waveform [B,1,T'] (vits.py:1175-1198)."""
        from .audio import wav_to_spec
        au = _get(self.config, "audio")
        if reference_wav.dim() == 2:
            reference_wav = reference_wav.unsqueeze(1)
        y = wav_to_spec(reference_wav, au.fft_size, au.hop_length, au.win_length, center=False)
        y_lengths = torch.tensor([y.size(-1)] * y.size(0)).to(y.device)
        speaker_cond_src = reference_speaker_id if reference_speaker_id is not None else reference_d_vector
        speaker_cond_tgt = speaker_id if speaker_id is not None else d_vector
        wav, _, _ = self.voice_conversion(y, y_lengths, speaker_cond_src, speaker_cond_tgt,
                                          posterior_noise=posterior_noise)
        return wav

    @torch.no_grad()
    def voice_conversion(self, y, y_lengths, speaker_cond_src, speaker_cond_tgt, *, posterior_noise=None):
        """y [B,C,T] linear spectrograms -> (o_hat, y_mask, (z, z_p, z_hat))   (vits.py:1200-1232).
        ``posterior_noise`` [B,H,T] replaces the posterior encoder's randn_like draw (networks.py:287)."""
        assert self.num_speakers > 0, "num_speakers have to be larger than 0."
        _lib.require_cuda(y, "y")
        a = self.args
        if a.use_speaker_embedding and not a.use_d_vector_file:
            ids = lambda v: torch.as_tensor(v, dtype=torch.int64, device=y.device).reshape(-1)
            g_src = self.emb_g(ids(speaker_cond_src)).unsqueeze(-1)
            g_tgt = self.emb_g(ids(speaker_cond_tgt)).unsqueeze(-1)
        elif not a.use_speaker_embedding and a.use_d_vector_file:
            g_src = F.normalize(speaker_cond_src.to(y.device)).unsqueeze(-1)
            g_tgt = F.normalize(speaker_cond_tgt.to(y.device)).unsqueeze(-1)
        else:
            raise RuntimeError(" [!] Voice conversion is only supported on multi-speaker models.")
        with _Stage(self, "posterior_encoder"):
            z, _, _, y_mask = self.posterior_encoder(y, y_lengths, g=g_src, noise=posterior_noise)
        with _Stage(self, "flow"):
            z_p = self.flow(z, y_mask, g=g_src)
            z_hat = self.flow(z_p, y_mask, g=g_tgt, reverse=True)
        with _Stage(self, "waveform_decoder"):
            o_hat = self.waveform_decoder(z_hat * y_mask, g=g_tgt)
        return o_hat, y_mask, (z, z_p, z_hat)

    def forward(self, *args, **kwargs):
        raise NotImplementedError("tts_b200.Vits implements the inference paths only "
                                  "(.inference, .voice_conversion); training is out of scope")

    # ------------------------------------------------------------------ checkpoints (vits.py:1698-1725)
    def load_checkpoint(self, config, checkpoint_path, eval=False, strict=True, cache=False):  # pylint: disable=redefined-builtin
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        model = {k: v for k, v in state["model"].items() if "speaker_encoder" not in k}
        model = {k: v for k, v in model.items() if not k.startswith("disc.")}  # training-only sub-module
        if hasattr(self, "emb_g") and model["emb_g.weight"].shape != self.emb_g.weight.shape:
            n_new = self.emb_g.weight.shape[0] - model["emb_g.weight"].shape[0]
            model["emb_g.weight"] = torch.cat([model["emb_g.weight"], torch.randn(n_new, model["emb_g.weight"].shape[1])], 0)
        self.load_state_dict(model, strict=strict)
        self.repack()      # packed device handles are rebuilt from the new weights on the next call
        if eval:
            self.eval()
            assert not self.training

    def load_fairseq_checkpoint(self, config, checkpoint_dir, eval=False, strict=True):  # pylint: disable=redefined-builtin
        """VITS checkpoints released by fairseq (MMS): ``config.json`` + ``G_100000.pth`` + ``vocab.txt``
        (vits.py:1727-1769): sets the sample rate, builds the character tokenizer from the vocabulary, resizes the
        text embedding to it and loads the re-keyed weights."""
        import json
        import os

        from .text import FairseqVocab, TTSTokenizer, basic_cleaners, rehash_fairseq_vits_checkpoint
        with open(os.path.join(checkpoint_dir, "config.json"), "r", encoding="utf-8") as f:
            config_org = json.load(f)
        _get(self.config, "audio").sample_rate = config_org["data"]["sampling_rate"]
        vocab = FairseqVocab(os.path.join(checkpoint_dir, "vocab.txt"))
        self.text_encoder.emb = nn.Embedding(vocab.num_chars, _get(config, "model_args").hidden_channels)
        self.text_encoder._cfg["n_vocab"] = vocab.num_chars
        self.tokenizer = TTSTokenizer(use_phonemes=False, text_cleaner=basic_cleaners, characters=vocab, phonemizer=None,
                                      add_blank=config_org["data"]["add_blank"], use_eos_bos=False)
        new_chk = rehash_fairseq_vits_checkpoint(os.path.join(checkpoint_dir, "G_100000.pth"))
        new_chk = {k: v for k, v in new_chk.items() if not k.startswith("disc.")}   # training-only sub-module
        self.load_state_dict(new_chk, strict=strict)
        self.repack()
        if eval:
            self.eval()
            assert not self.training

    def repack(self):
        for m in self.modules():
            if isinstance(m, EngineModule) and m is not self:
                m._drop_handle()
        self.waveform_decoder.repack()
