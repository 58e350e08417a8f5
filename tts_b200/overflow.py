"""Drop-in for the inference path of TTS.tts.models.overflow.Overflow (TTS/tts/models/overflow.py:24-401) and
TTS.tts.models.neuralhmm_tts.NeuralhmmTTS, with the model-side fields of their configs
(TTS/tts/configs/overflow_config.py, neuralhmm_tts_config.py), on sm_90a kernels.

``inference`` runs in one library handle: the encoder (embedding, conv + BatchNorm blocks, bidirectional LSTM), the
autoregressive neural-HMM sampling loop on the device (CUDA graph chunks of frames, one small host read per chunk),
and for Overflow the Glow decoder in reverse.  ``model_outputs`` ``[B, T, 80]`` feeds ``tts_b200.vocoder.vocoder_input``
and a HiFiGAN vocoder directly.

Kept surface: ``Overflow`` / ``NeuralhmmTTS(config, ap, tokenizer, speaker_manager)``, ``init_from_config``,
``inference(text, aux_input)`` with the ``aux_input`` keys ``x_lengths``, ``sampling_temp``, ``max_sampling_time`` and
``duration_threshold``, ``load_checkpoint(config, path, eval)``, ``update_mean_std``, ``normalize`` /
``inverse_normalize`` and the reference ``state_dict`` keys (including ``mean`` / ``std`` and ``neural_hmm.go_tokens``).

Differences from the reference, on purpose:

1. Batched, per row.  The reference's ``Encoder.inference`` ignores ``x_lengths`` (no packing), so in a padded batch
   its backward LSTM starts from the pad tokens.  Here row b equals the reference's
   ``inference(text[b:b+1, :x_lengths[b]])``; at B = 1 without padding it is the reference call.
2. Random draws.  The reference draws the emission noise and the prenet dropout masks with several small generator
   calls per frame and row.  Here they are drawn in bulk on the device, from torch's generator for that device, before
   the loop.  ``inference`` also takes them as the keyword argument ``draws`` (an addition to the reference signature):
   ``{"noise": [B, max_sampling_time, C] standard-normal, "dropout": [B, max_sampling_time, prenet_n_layers,
   prenet_dim] bool (True keeps a unit)}``; the emission sample is ``mean + (std * sampling_temp) * noise``.

``input_parameters`` / ``output_parameters`` (plotting traces of the reference) are returned as ``None``.
``max_sampling_time`` must be >= 1 (the reference's 0, "no limit", has no bound for the output buffers).
Training (``forward``), ``prenet_type="bn"``, speaker conditioning and ``deterministic_transition=False`` raise
``NotImplementedError``.
"""
import ctypes
from dataclasses import asdict, dataclass, field
from typing import List

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from .glow_tts import _CouplingBlock, _Decoder, _InvConvNear
from .layers import EngineModule, _host

CHUNK_FRAMES = 32     # frames per CUDA graph replay (one host read per chunk)


class _ConfigBase:
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


@dataclass
class NeuralhmmTTSConfig(_ConfigBase):
    """The model-side fields of TTS/tts/configs/neuralhmm_tts_config.py with the reference defaults."""
    model: str = "NeuralHMM_TTS"
    force_generate_statistics: bool = False
    mel_statistics_parameter_path: str = None
    num_chars: int = None
    state_per_phone: int = 2
    encoder_in_out_features: int = 512
    encoder_n_convolutions: int = 3
    out_channels: int = 80
    ar_order: int = 1
    sampling_temp: float = 0
    deterministic_transition: bool = True
    duration_threshold: float = 0.43
    use_grad_checkpointing: bool = True
    max_sampling_time: int = 1000
    prenet_type: str = "original"
    prenet_dim: int = 256
    prenet_n_layers: int = 2
    prenet_dropout: float = 0.5
    prenet_dropout_at_inference: bool = True
    memory_rnn_dim: int = 1024
    outputnet_size: List[int] = field(default_factory=lambda: [1024])
    flat_start_params: dict = field(default_factory=lambda: {"mean": 0.0, "std": 1.0, "transition_p": 0.14})
    std_floor: float = 0.001
    r: int = 1
    use_d_vector_file: bool = False
    use_speaker_embedding: bool = False


@dataclass
class OverflowConfig(_ConfigBase):
    """The model-side fields of TTS/tts/configs/overflow_config.py with the reference defaults."""
    model: str = "Overflow"
    force_generate_statistics: bool = False
    mel_statistics_parameter_path: str = None
    num_chars: int = None
    state_per_phone: int = 2
    encoder_in_out_features: int = 512
    encoder_n_convolutions: int = 3
    out_channels: int = 80
    ar_order: int = 1
    sampling_temp: float = 0.334
    deterministic_transition: bool = True
    duration_threshold: float = 0.55
    use_grad_checkpointing: bool = True
    max_sampling_time: int = 1000
    prenet_type: str = "original"
    prenet_dim: int = 256
    prenet_n_layers: int = 2
    prenet_dropout: float = 0.5
    prenet_dropout_at_inference: bool = False
    memory_rnn_dim: int = 1024
    outputnet_size: List[int] = field(default_factory=lambda: [1024])
    flat_start_params: dict = field(default_factory=lambda: {"mean": 0.0, "std": 1.0, "transition_p": 0.14})
    std_floor: float = 0.01
    hidden_channels_dec: int = 150
    kernel_size_dec: int = 5
    dilation_rate: int = 1
    num_flow_blocks_dec: int = 12
    num_block_layers: int = 4
    dropout_p_dec: float = 0.05
    num_splits: int = 4
    num_squeeze: int = 2
    sigmoid_scale: bool = False
    c_in_channels: int = 0
    r: int = 1
    use_d_vector_file: bool = False
    use_speaker_embedding: bool = False


# ----------------------------------------------------------------------------- parameter containers
class _ConvBNBlock(nn.Module):
    """Parameters of TTS/tts/layers/tacotron/tacotron2.py:11-44 (activation "relu")."""

    def __init__(self, channels, kernel_size):
        super().__init__()
        self.convolution1d = nn.Conv1d(channels, channels, kernel_size, padding=(kernel_size - 1) // 2)
        self.batch_normalization = nn.BatchNorm1d(channels, momentum=0.1, eps=1e-5)


class _Encoder(nn.Module):
    """Parameters of TTS/tts/layers/overflow/common_layers.py:12-42."""

    def __init__(self, num_chars, state_per_phone, in_out_channels=512, n_convolutions=3):
        super().__init__()
        self.state_per_phone, self.in_out_channels = state_per_phone, in_out_channels
        self.emb = nn.Embedding(num_chars, in_out_channels)
        self.convolutions = nn.ModuleList([_ConvBNBlock(in_out_channels, 5) for _ in range(n_convolutions)])
        self.lstm = nn.LSTM(in_out_channels, int(in_out_channels / 2) * state_per_phone, num_layers=1,
                            batch_first=True, bias=True, bidirectional=True)


class _Linear(nn.Module):
    """Parameters of TTS/tts/layers/tacotron/common_layers.py:6-25."""

    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.linear_layer = nn.Linear(in_features, out_features, bias=bias)
        nn.init.xavier_uniform_(self.linear_layer.weight, gain=nn.init.calculate_gain("linear"))


class _Prenet(nn.Module):
    """Parameters of TTS/tts/layers/tacotron/common_layers.py:63-107 (prenet_type "original", bias=False)."""

    def __init__(self, in_features, out_features):
        super().__init__()
        ins = [in_features] + out_features[:-1]
        self.linear_layers = nn.ModuleList([_Linear(i, o, bias=False) for i, o in zip(ins, out_features)])


class _ParameterModel(nn.Module):
    """Parameters of TTS/tts/layers/overflow/common_layers.py:95-131, flat-start output layer included."""

    def __init__(self, outputnet_size, input_size, output_size, frame_channels, flat_start_params):
        super().__init__()
        self.layers = nn.ModuleList([_Linear(i, o) for i, o in zip([input_size] + outputnet_size[:-1], outputnet_size)])
        self.last_layer = nn.Linear(outputnet_size[-1], output_size)
        with torch.no_grad():
            self.last_layer.weight.zero_()
            fc = frame_channels
            self.last_layer.bias[0:fc] = flat_start_params["mean"]
            self.last_layer.bias[fc:2 * fc] = torch.log(torch.clamp(torch.exp(torch.tensor(
                float(flat_start_params["std"]))) - 1.0, min=1e-4))
            tp = torch.tensor(float(flat_start_params["transition_p"]))
            self.last_layer.bias[2 * fc:] = torch.log(torch.clamp(tp / (1.0 - tp), min=1e-4))


class _Outputnet(nn.Module):
    def __init__(self, encoder_dim, memory_rnn_dim, frame_channels, outputnet_size, flat_start_params):
        super().__init__()
        self.parametermodel = _ParameterModel(outputnet_size, memory_rnn_dim + encoder_dim, 2 * frame_channels + 1,
                                              frame_channels, flat_start_params)


class _NeuralHMM(nn.Module):
    """Parameters of TTS/tts/layers/overflow/neural_hmm.py:48-92."""

    def __init__(self, frame_channels, ar_order, encoder_dim, prenet_dim, prenet_n_layers, memory_rnn_dim,
                 outputnet_size, flat_start_params):
        super().__init__()
        assert ar_order > 0, f"AR order must be greater than 0 provided {ar_order}"
        self.prenet = _Prenet(frame_channels * ar_order, [prenet_dim] * prenet_n_layers)
        self.memory_rnn = nn.LSTMCell(input_size=prenet_dim, hidden_size=memory_rnn_dim)
        self.output_net = _Outputnet(encoder_dim, memory_rnn_dim, frame_channels, outputnet_size, flat_start_params)
        self.register_buffer("go_tokens", torch.zeros(ar_order, 1))


class _OverflowDecoder(nn.Module):
    """Parameters of TTS/tts/layers/overflow/decoder.py:8-54 (a Glow decoder)."""

    def __init__(self, in_channels, hidden_channels, kernel_size, dilation_rate, num_flow_blocks, num_coupling_layers,
                 dropout_p=0.0, num_splits=4, num_squeeze=2):
        super().__init__()
        self.glow_decoder = _Decoder(in_channels, hidden_channels, kernel_size, dilation_rate, num_flow_blocks,
                                     num_coupling_layers, dropout_p, num_splits, num_squeeze, 0)

    def store_inverse(self):
        for f in self.glow_decoder.flows:
            if isinstance(f, (_InvConvNear, _CouplingBlock)):
                f.store_inverse()


def _format_aux_input(defaults, aux_input):
    """TTS/utils/generic_utils.py format_aux_input: a missing or None entry takes the default."""
    out = dict(aux_input or {})
    for k, v in defaults.items():
        if out.get(k, None) is None:
            out[k] = v
    return out


# ----------------------------------------------------------------------------- models
class NeuralhmmTTS(EngineModule):
    """Neural-HMM text -> mel synthesiser (no decoder), inference path on sm_90a kernels."""

    _destroy = "b200tts_overflow_destroy"
    _has_decoder = False

    def __init__(self, config, ap=None, tokenizer=None, speaker_manager=None):
        super().__init__()
        self.config, self.ap, self.tokenizer, self.speaker_manager = config, ap, tokenizer, speaker_manager
        for key in config:
            setattr(self, key, config[key])
        if tokenizer is not None:   # BaseTTS._set_model_args (base_tts.py:61-66)
            self.num_chars = tokenizer.characters.num_chars
        self.decoder_output_dim = self.out_channels
        self.encoder = _Encoder(self.num_chars, self.state_per_phone, self.encoder_in_out_features,
                                self.encoder_n_convolutions)
        self.neural_hmm = _NeuralHMM(self.out_channels, self.ar_order, self.encoder_in_out_features, self.prenet_dim,
                                     self.prenet_n_layers, self.memory_rnn_dim, self.outputnet_size,
                                     self.flat_start_params)
        if self._has_decoder:
            self.decoder = _OverflowDecoder(self.out_channels, self.hidden_channels_dec, self.kernel_size_dec,
                                            self.dilation_rate, self.num_flow_blocks_dec, self.num_block_layers,
                                            self.dropout_p_dec, self.num_splits, self.num_squeeze)
        self.register_buffer("mean", torch.tensor(0))
        self.register_buffer("std", torch.tensor(1))

    @classmethod
    def init_from_config(cls, config, samples=None, verbose=True):  # pylint: disable=unused-argument
        """overflow.py:252-266 without the host-side managers (tokenizer / AudioProcessor are built by the caller)."""
        return cls(config)

    def update_mean_std(self, statistics_dict):
        self.mean.data = torch.tensor(statistics_dict["mean"])
        self.std.data = torch.tensor(statistics_dict["std"])
        self._drop_handle()

    def normalize(self, x):
        return x.sub(self.mean).div(self.std)

    def inverse_normalize(self, x):
        return x.mul(self.std).add(self.mean)

    # ------------------------------------------------------------------ packing
    def _check_supported(self):
        if self.prenet_type != "original":
            raise NotImplementedError("tts_b200: prenet_type 'bn' is not built (prenet_type 'original' only)")
        if not self.deterministic_transition:
            raise NotImplementedError("tts_b200: deterministic_transition=False (a multinomial draw per frame) is not "
                                      "built; the released models use the deterministic rule")
        if getattr(self, "c_in_channels", 0) or self.use_speaker_embedding or self.use_d_vector_file:
            raise NotImplementedError("tts_b200: speaker conditioning is not built for Overflow / Neural-HMM")
        if len(self.outputnet_size) > 8 or self.prenet_n_layers > 8 or self.encoder_n_convolutions > 8:
            raise NotImplementedError("tts_b200: at most 8 prenet, output-net and encoder conv layers")

    def _create(self, device):
        self._check_supported()
        e, h = self.encoder, self.neural_hmm
        c = self.out_channels
        sizes = (ctypes.c_int * 8)(*(list(self.outputnet_size) + [0] * (8 - len(self.outputnet_size))))
        dec = [self.hidden_channels_dec, self.kernel_size_dec, self.dilation_rate, self.num_flow_blocks_dec,
               self.num_block_layers, self.num_splits, self.num_squeeze, int(self.sigmoid_scale)] \
            if self._has_decoder else [0] * 8
        cfg = _lib.OverflowConfigC(self.num_chars, self.encoder_in_out_features, self.encoder_n_convolutions,
                              self.state_per_phone, c, self.ar_order, self.prenet_dim, self.prenet_n_layers,
                              int(bool(self.prenet_dropout)), self.memory_rnn_dim, len(self.outputnet_size), sizes,
                              float(self.std_floor), int(self._has_decoder), *dec)
        t = [_host(e.emb.weight)]
        for blk in e.convolutions:
            bn = blk.batch_normalization
            t += [_host(blk.convolution1d.weight), _host(blk.convolution1d.bias), _host(bn.weight), _host(bn.bias),
                  _host(bn.running_mean), _host(bn.running_var)]
        for sfx in ("", "_reverse"):
            t += [_host(getattr(e.lstm, f"{n}_l0{sfx}")) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        t += [_host(h.go_tokens.reshape(-1))]
        t += [_host(lin.linear_layer.weight) for lin in h.prenet.linear_layers]
        m = h.memory_rnn
        t += [_host(m.weight_ih), _host(m.weight_hh), _host(m.bias_ih), _host(m.bias_hh)]
        pm = h.output_net.parametermodel
        for lin in pm.layers:
            t += [_host(lin.linear_layer.weight), _host(lin.linear_layer.bias)]
        t += [_host(pm.last_layer.weight), _host(pm.last_layer.bias)]
        t += [_host(self.mean.to(torch.float32).expand(c)), _host(self.std.to(torch.float32).expand(c))]
        if self._has_decoder:
            for n in range(self.num_flow_blocks_dec):
                fl = self.decoder.glow_decoder.flows
                an, ic, cb = fl[3 * n], fl[3 * n + 1], fl[3 * n + 2]
                t += [_host(an.logs.reshape(-1)), _host(an.bias.reshape(-1)), ic.inverse().contiguous()]
                t += [_host(cb.start.weight), _host(cb.start.bias)] + cb.wn.ordered_weights() + \
                     [_host(cb.end.weight), _host(cb.end.bias)]
        return self._make("b200tts_overflow_create", cfg, t)

    # ------------------------------------------------------------------ inference
    def _draws(self, b, max_t, temp, dropout, draws, dev):
        c, pdim, nl = self.out_channels, self.prenet_dim, self.prenet_n_layers
        draws = draws or {}
        noise = drop = None
        if temp > 0:
            noise = draws.get("noise", None)
            noise = torch.randn((b, max_t, c), device=dev) if noise is None else noise.to(dev, torch.float32)
            if noise.shape[0] != b or noise.shape[2] != c or noise.shape[1] < max_t:
                raise ValueError(f"tts_b200: draws['noise'] must be [{b}, >= {max_t}, {c}], got {tuple(noise.shape)}")
            noise = noise[:, :max_t].contiguous()
        if dropout:
            drop = draws.get("dropout", None)
            if drop is None:
                drop = torch.empty((b, max_t, nl, pdim), dtype=torch.uint8, device=dev).bernoulli_(0.5)
            else:
                if drop.shape[0] != b or drop.shape[1] < max_t or tuple(drop.shape[2:]) != (nl, pdim):
                    raise ValueError(f"tts_b200: draws['dropout'] must be [{b}, >= {max_t}, {nl}, {pdim}], "
                                     f"got {tuple(drop.shape)}")
                drop = drop[:, :max_t].to(dev, torch.uint8).contiguous()
        return noise, drop

    @torch.no_grad()
    def inference(self, text, aux_input={"x_lengths": None, "sampling_temp": None, "max_sampling_time": None,
                                         "duration_threshold": None}, *, draws=None):  # pylint: disable=dangerous-default-value
        """text int64 [B, T] (CUDA) -> dict(model_outputs [B, T', C], model_outputs_len, alignments
        [B, T_hmm + 1, N_max + 1], hmm_outputs [B, T_hmm, C], hmm_outputs_len, input_parameters None,
        output_parameters None).  ``draws`` (optional): the emission noise and prenet dropout masks, see the module
        docstring.  One host read per chunk of 32 frames drives the loop."""
        self._check_supported()
        _lib.require_cuda(text, "text")
        dev = text.device
        tok = text.to(torch.int64).contiguous()
        b, tt = tok.shape
        aux = _format_aux_input({"x_lengths": torch.sum(text != 0, dim=1), "sampling_temp": self.sampling_temp,
                                 "max_sampling_time": self.max_sampling_time,
                                 "duration_threshold": self.duration_threshold}, aux_input)
        x_lengths = aux["x_lengths"]
        lens = x_lengths.to(device=dev, dtype=torch.int64).contiguous()
        max_t = int(aux["max_sampling_time"] or 0)
        if max_t < 1:
            raise ValueError("tts_b200: max_sampling_time must be >= 1 (0, no limit, is not supported)")
        if b == 0:
            raise ValueError("tts_b200: empty batch")
        if int(lens.min()) < 1 or int(lens.max()) > tt:
            raise ValueError(f"tts_b200: x_lengths must be in [1, {tt}]")
        temp = float(aux["sampling_temp"])
        thr = float(aux["duration_threshold"])
        dropout = bool(self.prenet_dropout) and (self.training or bool(self.prenet_dropout_at_inference))
        noise, drop = self._draws(b, max_t, temp, dropout, draws, dev)
        c, e, spp = self.out_channels, self.encoder_in_out_features, self.state_per_phone
        f32 = dict(dtype=torch.float32, device=dev)
        states = torch.empty((b, tt * spp, e), **f32)
        hmm = torch.empty((b, max_t, c), **f32)
        st_tr = torch.empty((b, max_t + 1), dtype=torch.int32, device=dev)
        frames = (ctypes.c_int32 * b)()
        h = self.handle(dev)
        L = _lib.lib()
        s = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            ws = _lib.workspace(dev, L.b200tts_overflow_workspace_bytes(h, b, tt, max_t), "overflow")
            wsp, wsn = _lib.ptr(ws), ctypes.c_size_t(ws.numel())
            _lib.check(L.b200tts_overflow_encode(h, _lib.ptr(tok), _lib.ptr(lens), b, tt, _lib.ptr(states), wsp, wsn, s),
                       "overflow_encode")
            _lib.check(L.b200tts_overflow_sample(h, _lib.ptr(lens), b, tt, ctypes.c_float(temp), max_t,
                                                 ctypes.c_float(thr), _lib.ptr(noise), _lib.ptr(drop), CHUNK_FRAMES,
                                                 _lib.ptr(hmm), _lib.ptr(st_tr), frames, wsp, wsn, s),
                       "overflow_sample")
            n_frames = torch.tensor(list(frames), dtype=torch.int32)
            f_max = int(n_frames.max())
            frames_dev = n_frames.to(dev)
            f_out = (f_max // self.num_squeeze) * self.num_squeeze if self._has_decoder else f_max
            mel = torch.empty((b, f_out, c), **f32)
            _lib.check(L.b200tts_overflow_decode(h, _lib.ptr(hmm), _lib.ptr(frames_dev), b, f_max, max_t,
                                                 _lib.ptr(mel), wsp, wsn, s), "overflow_decode")
        hmm_len = n_frames.to(device=dev, dtype=x_lengths.dtype)
        st = st_tr[:, :f_max + 1].to(torch.int64)
        width = int(st.max()) + 1
        align = F.one_hot(st.clamp(min=0), width) * (st >= 0).unsqueeze(-1)
        out_len = torch.div(hmm_len, self.num_squeeze, rounding_mode="floor") * self.num_squeeze \
            if self._has_decoder else hmm_len
        return {"hmm_outputs": hmm[:, :f_max], "hmm_outputs_len": hmm_len, "alignments": align,
                "input_parameters": None, "output_parameters": None, "model_outputs": mel,
                "model_outputs_len": out_len}

    # ------------------------------------------------------------------ out of scope
    def forward(self, *args, **kwargs):
        raise NotImplementedError("tts_b200: Overflow / Neural-HMM implement inference only; training (forward, the "
                                  "HMM forward algorithm) is out of scope")

    # ------------------------------------------------------------------ checkpoints (overflow.py load_checkpoint)
    def load_checkpoint(self, config, checkpoint_path, eval=False, strict=True, cache=False):  # pylint: disable=unused-argument, redefined-builtin
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        self.load_state_dict(state["model"])
        self._drop_handle()
        if eval:
            self.eval()
            if self._has_decoder:
                self.decoder.store_inverse()
            assert not self.training

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # mean / std are scalars until update_mean_std makes them per-channel: take the checkpoint's shape
        for k in ("mean", "std"):
            v = state_dict.get(prefix + k, None)
            if v is not None and getattr(self, k).shape != v.shape:
                setattr(self, k, torch.empty_like(v))
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


class Overflow(NeuralhmmTTS):
    """Overflow text -> mel synthesiser (neural HMM + Glow decoder), inference path on sm_90a kernels."""

    _has_decoder = True
