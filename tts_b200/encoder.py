"""Drop-in for the H/ASP speaker encoder: TTS.encoder.models.resnet.ResNetSpeakerEncoder
(/root/reference/TTS/encoder/models/resnet.py:59-198, base_encoder.py:25-161) and
TTS.encoder.utils.generic_utils.setup_encoder_model (generic_utils.py:118-136).

Same constructor, same ``state_dict`` keys (the torch modules below are only parameter containers, including the
``torch_spec`` front-end buffers and every ``num_batches_tracked``), so reference checkpoints load strictly.  The
arithmetic -- pre-emphasis, mel spectrogram, instance norm, the SE-ResNet trunk, attentive statistics pooling, the
projection, the l2 norm and the mean over windows -- runs in libtts_b200.so (b200tts_speaker_encoder_forward); there
is no PyTorch fallback.  torchaudio is not a dependency: the default Hamming window and HTK mel filterbank are built
here, and a loaded checkpoint's buffers replace them.
"""
import ctypes
import math

import numpy as np
import torch
from torch import nn

from . import _lib


def htk_mel_filterbank(n_freqs, f_min, f_max, n_mels, sample_rate):
    """[n_freqs, n_mels] triangular filters on the HTK mel scale without area normalisation (torchaudio's
    ``melscale_fbanks(..., norm=None, mel_scale="htk")``), computed in float32 in the same order."""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_min = 2595.0 * math.log10(1.0 + (f_min / 700.0))
    m_max = 2595.0 * math.log10(1.0 + (f_max / 700.0))
    m_pts = torch.linspace(m_min, m_max, n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.max(torch.zeros(1), torch.min(down, up))


class _PreEmphasis(nn.Module):
    """Key layout of base_encoder.PreEmphasis: buffer ``filter`` [1, 1, 2] = (-coefficient, 1)."""

    def __init__(self, coefficient=0.97):
        super().__init__()
        self.coefficient = coefficient
        self.register_buffer("filter", torch.FloatTensor([-coefficient, 1.0]).unsqueeze(0).unsqueeze(0))


class _Spectrogram(nn.Module):
    def __init__(self, win_length):
        super().__init__()
        self.register_buffer("window", torch.hamming_window(win_length))


class _MelScale(nn.Module):
    def __init__(self, n_mels, sample_rate, n_freqs):
        super().__init__()
        self.register_buffer("fb", htk_mel_filterbank(n_freqs, 0.0, float(sample_rate // 2), n_mels, sample_rate))


class _MelSpectrogram(nn.Module):
    """Key layout of torchaudio.transforms.MelSpectrogram: ``spectrogram.window``, ``mel_scale.fb``."""

    def __init__(self, sample_rate, n_fft, win_length, hop_length, n_mels):
        super().__init__()
        self.sample_rate, self.n_fft, self.win_length, self.hop_length, self.n_mels = (
            sample_rate, n_fft, win_length, hop_length, n_mels)
        self.spectrogram = _Spectrogram(win_length)
        self.mel_scale = _MelScale(n_mels, sample_rate, n_fft // 2 + 1)


class _SELayer(nn.Module):
    def __init__(self, channel, reduction=8):
        super().__init__()
        self.fc = nn.Sequential(nn.Linear(channel, channel // reduction), nn.ReLU(inplace=True),
                                nn.Linear(channel // reduction, channel), nn.Sigmoid())


class _SEBasicBlock(nn.Module):
    def __init__(self, inplanes, planes, stride=1, downsample=None, reduction=8):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.se = _SELayer(planes, reduction)
        self.downsample = downsample


def _bn(m):
    return [m.weight, m.bias, m.running_mean, m.running_var]


class ResNetSpeakerEncoder(nn.Module):
    # pylint: disable=dangerous-default-value
    def __init__(self, input_dim=64, proj_dim=512, layers=[3, 4, 6, 3], num_filters=[32, 64, 128, 256],
                 encoder_type="ASP", log_input=False, use_torch_spec=False, audio_config=None):
        super().__init__()
        if encoder_type not in ("ASP", "SAP"):
            raise ValueError("Undefined encoder")
        self.encoder_type = encoder_type
        self.input_dim = input_dim
        self.log_input = log_input
        self.use_torch_spec = use_torch_spec
        self.audio_config = audio_config
        self.proj_dim = proj_dim
        self._layers, self._filters = list(layers), list(num_filters)

        self.conv1 = nn.Conv2d(1, num_filters[0], kernel_size=3, stride=1, padding=1)
        self.relu = nn.ReLU(inplace=True)
        self.bn1 = nn.BatchNorm2d(num_filters[0])
        self.inplanes = num_filters[0]
        self.layer1 = self._create_layer(num_filters[0], layers[0])
        self.layer2 = self._create_layer(num_filters[1], layers[1], stride=(2, 2))
        self.layer3 = self._create_layer(num_filters[2], layers[2], stride=(2, 2))
        self.layer4 = self._create_layer(num_filters[3], layers[3], stride=(2, 2))
        self.instancenorm = nn.InstanceNorm1d(input_dim)
        if self.use_torch_spec:
            a = audio_config
            self.torch_spec = nn.Sequential(
                _PreEmphasis(a["preemphasis"]),
                _MelSpectrogram(a["sample_rate"], a["fft_size"], a["win_length"], a["hop_length"], a["num_mels"]))
        else:
            self.torch_spec = None
        outmap_size = int(self.input_dim / 8)
        self.attention = nn.Sequential(
            nn.Conv1d(num_filters[3] * outmap_size, 128, kernel_size=1), nn.ReLU(), nn.BatchNorm1d(128),
            nn.Conv1d(128, num_filters[3] * outmap_size, kernel_size=1), nn.Softmax(dim=2))
        out_dim = num_filters[3] * outmap_size * (2 if encoder_type == "ASP" else 1)
        self.fc = nn.Linear(out_dim, proj_dim)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        self._handle = None
        self._handle_device = None
        # a parent's load_state_dict recurses through _load_from_state_dict, so the packed handle is dropped from a hook
        self._register_load_state_dict_pre_hook(lambda *a, **k: self._drop_handle())

    def _create_layer(self, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes:
            downsample = nn.Sequential(nn.Conv2d(self.inplanes, planes, kernel_size=1, stride=stride, bias=False),
                                       nn.BatchNorm2d(planes))
        layers = [_SEBasicBlock(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes
        layers += [_SEBasicBlock(planes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    # ------------------------------------------------------------------ handle
    def _drop_handle(self):
        if getattr(self, "_handle", None) is not None:
            _lib.lib().b200tts_speaker_encoder_destroy(self._handle)
        self._handle = None

    def __del__(self):
        try:
            self._drop_handle()
        except Exception:  # pylint: disable=broad-except
            pass

    def _apply(self, fn, *a, **kw):
        self._drop_handle()
        return super()._apply(fn, *a, **kw)

    def _ordered_weights(self):
        """Host tensors in the order of b200tts_speaker_encoder_create (include/tts_b200.h)."""
        w = []
        if self.use_torch_spec:
            pre, mel = self.torch_spec[0], self.torch_spec[1]
            w += [pre.filter.reshape(-1), mel.spectrogram.window, mel.mel_scale.fb]
        w += [self.conv1.weight, self.conv1.bias] + _bn(self.bn1)
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            for blk in layer:
                w += [blk.conv1.weight] + _bn(blk.bn1) + [blk.conv2.weight] + _bn(blk.bn2)
                w += [blk.se.fc[0].weight, blk.se.fc[0].bias, blk.se.fc[2].weight, blk.se.fc[2].bias]
                if blk.downsample is not None:
                    w += [blk.downsample[0].weight] + _bn(blk.downsample[1])
        a = self.attention
        w += [a[0].weight, a[0].bias] + _bn(a[2]) + [a[3].weight, a[3].bias, self.fc.weight, self.fc.bias]
        return [t.detach().to("cpu", torch.float32).contiguous() for t in w]

    def _ensure_handle(self, device):
        if self._handle is not None and self._handle_device == device:
            return self._handle
        self._drop_handle()
        cfg = _lib.SpeakerEncoderConfigC()
        cfg.input_dim, cfg.proj_dim = self.input_dim, self.proj_dim
        for i in range(4):
            cfg.layers[i], cfg.num_filters[i] = self._layers[i], self._filters[i]
        cfg.encoder_type = 1 if self.encoder_type == "ASP" else 0
        cfg.log_input, cfg.use_torch_spec = int(bool(self.log_input)), int(bool(self.use_torch_spec))
        if self.use_torch_spec:
            mel = self.torch_spec[1]
            cfg.fft_size, cfg.win_length, cfg.hop_length = mel.n_fft, mel.win_length, mel.hop_length
            if mel.spectrogram.window.numel() != mel.win_length or tuple(mel.mel_scale.fb.shape) != (
                    mel.n_fft // 2 + 1, self.input_dim):
                raise ValueError("tts_b200.ResNetSpeakerEncoder: front-end buffers do not match the audio config")
        ws = self._ordered_weights()
        arr = (ctypes.c_void_p * len(ws))(*[t.data_ptr() for t in ws])
        out = ctypes.c_void_p()
        with torch.cuda.device(device):
            rc = _lib.lib().b200tts_speaker_encoder_create(ctypes.byref(cfg), arr, len(ws), ctypes.byref(out))
        _lib.check(rc, "speaker_encoder_create")
        self._handle, self._handle_device = out, device
        return out

    # ------------------------------------------------------------------ launches
    def _run(self, flat, starts, win_len, groups, l2_norm, stage=None):
        """Windows ``flat[starts[b] : ...]`` of ``win_len`` samples (or [input_dim, win_len] frames) -> [groups, proj]
        (or the dense features of ``stage``)."""
        dev = flat.device
        h = self._ensure_handle(dev)
        L = _lib.lib()
        st = torch.as_tensor(starts, dtype=torch.int32).to(dev)
        b = int(st.numel())
        with torch.cuda.device(dev):
            nbytes = L.b200tts_speaker_encoder_workspace_bytes(h, b, win_len)
            ws = _lib.workspace(dev, nbytes, "speaker_encoder")
            if stage is None:
                out = torch.empty((groups, self.proj_dim), dtype=torch.float32, device=dev)
                rc = L.b200tts_speaker_encoder_forward(h, _lib.ptr(flat), _lib.ptr(st), b, win_len, groups, int(l2_norm),
                                                       _lib.ptr(out), _lib.ptr(ws), ctypes.c_size_t(ws.numel()),
                                                       _lib.stream_ptr(dev))
                _lib.check(rc, "speaker_encoder_forward")
                return out
            shape = self.feature_shape(b, win_len, stage)
            out = torch.empty(shape, dtype=torch.float32, device=dev)
            rc = L.b200tts_speaker_encoder_features(h, _lib.ptr(flat), _lib.ptr(st), b, win_len, stage, _lib.ptr(out),
                                                    _lib.ptr(ws), ctypes.c_size_t(ws.numel()), _lib.stream_ptr(dev))
            _lib.check(rc, "speaker_encoder_features")
            return out

    def feature_shape(self, batch, win_len, stage):
        """Shape of ``forward_features(x, stage)`` for ``batch`` windows of ``win_len`` samples / frames."""
        t = win_len // self.torch_spec[1].hop_length + 1 if self.use_torch_spec else win_len
        if stage == 0:
            return (batch, self.input_dim, t)
        h = self.input_dim
        for _ in range(1, stage):
            t, h = (t + 1) // 2, (h + 1) // 2
        return (batch, self._filters[stage - 1], h, t)

    def _windows(self, x):
        """x [N, 1, T] / [N, T] waveforms or [N, input_dim, T] spectrograms -> (flat, starts, window length)."""
        _lib.require_cuda(x, "x")
        x = x.to(torch.float32)
        if self.use_torch_spec:
            x = x.reshape(x.shape[0], -1).contiguous()
            n, t = x.shape
            return x.reshape(-1), [i * t for i in range(n)], t
        if x.ndim != 3 or x.shape[1] != self.input_dim:
            raise ValueError(f"tts_b200.ResNetSpeakerEncoder: expected [N, {self.input_dim}, T] spectrograms, "
                             f"got {tuple(x.shape)}")
        x = x.contiguous()
        n, d, t = x.shape
        return x.reshape(-1), [i * d * t for i in range(n)], t

    @torch.no_grad()
    def forward(self, x, l2_norm=False):
        """x [N, 1, T] waveform (``use_torch_spec``) or [N, input_dim, T] spectrogram -> [N, proj_dim] (resnet.py:153)."""
        flat, starts, t = self._windows(x)
        return self._run(flat, starts, t, len(starts), l2_norm)

    @torch.no_grad()
    def forward_features(self, x, stage):
        """The activations after ``stage`` (0: the instance-normed input [N, input_dim, T']; 1..4: the output of
        ``layer<stage>``, [N, C, H, T]) for the same input as ``forward``."""
        flat, starts, t = self._windows(x)
        return self._run(flat, starts, t, 1, False, stage=int(stage))

    @torch.no_grad()
    def inference(self, x, l2_norm=True):
        return self.forward(x, l2_norm)

    def _window_plan(self, n_rows, row_len, num_frames, num_eval):
        """compute_embedding's windows (base_encoder.py:68-96): (window length, [start of each window])."""
        if self.use_torch_spec:
            num_frames = num_frames * self.audio_config["hop_length"]
        max_len = row_len
        if max_len < num_frames:
            num_frames = max_len
        offsets = np.linspace(0, max_len - num_frames, num=num_eval)
        return num_frames, [int(o) for o in offsets]

    @torch.no_grad()
    def compute_embedding(self, x, num_frames=250, num_eval=10, return_mean=True, l2_norm=True):
        """x [1, T] waveform (or [1, input_dim, T] spectrogram) -> [1, proj_dim] mean of ``num_eval`` window embeddings
        (``[num_eval, proj_dim]`` without ``return_mean``), base_encoder.py:67-96.  With spectrogram input the
        reference's ``max_len = x.shape[1]`` is the mel axis, so every window is the whole input."""
        _lib.require_cuda(x, "x")
        x = x.to(torch.float32).contiguous()
        n = x.shape[0]
        nf, offsets = self._window_plan(n, x.shape[1], num_frames, num_eval)
        if self.use_torch_spec:
            if x.ndim != 2:
                raise ValueError(f"tts_b200.ResNetSpeakerEncoder.compute_embedding: expected [N, T], got {tuple(x.shape)}")
            t = x.shape[1]
            starts = [o + r * t for o in offsets for r in range(n)]
            win = nf
        else:
            if x.ndim != 3 or nf != self.input_dim:
                raise ValueError("tts_b200.ResNetSpeakerEncoder.compute_embedding: spectrogram windows must span "
                                 f"{self.input_dim} mel bins, got {tuple(x.shape)} -> {nf}")
            d, t = x.shape[1], x.shape[2]
            starts = [o * t + r * d * t for o in offsets for r in range(n)]
            win = t
        return self._run(x.reshape(-1), starts, win, 1 if return_mean else len(starts), l2_norm)

    @torch.no_grad()
    def compute_embeddings(self, wavs, num_frames=250, num_eval=10, l2_norm=True, max_clips_per_launch=64):
        """Batched ``compute_embedding`` for N waveforms at the encoder's sample rate (1-D or [1, T] CUDA tensors):
        returns [N, proj_dim], row i equal to ``compute_embedding(wavs[i].view(1, -1), num_frames, num_eval)`` up to
        the rounding of a different batch.  Clips of at least ``num_frames * hop_length`` samples share one window
        length and run together; shorter clips are grouped by exact length (the instance norm, SE and pooling reduce
        over the whole window, so windows of one length batch exactly)."""
        if not self.use_torch_spec:
            raise ValueError("tts_b200.ResNetSpeakerEncoder.compute_embeddings: takes waveforms (use_torch_spec=True)")
        clips = [_lib.require_cuda(w, "wavs[i]").reshape(-1) for w in wavs]
        if not clips:
            return torch.empty((0, self.proj_dim), dtype=torch.float32)
        dev = clips[0].device
        out = torch.empty((len(clips), self.proj_dim), dtype=torch.float32, device=dev)
        groups = {}
        for i, c in enumerate(clips):
            nf, offsets = self._window_plan(1, int(c.numel()), num_frames, num_eval)
            groups.setdefault(nf, []).append((i, offsets))
        for nf, members in groups.items():
            for k in range(0, len(members), max_clips_per_launch):
                part = members[k:k + max_clips_per_launch]
                flat = torch.cat([clips[i].to(device=dev, dtype=torch.float32) for i, _ in part])
                starts, base = [], 0
                for i, offsets in part:
                    starts += [base + o for o in offsets]
                    base += int(clips[i].numel())
                emb = self._run(flat, starts, nf, len(part), l2_norm)
                out[torch.tensor([i for i, _ in part], device=dev)] = emb
        return out

    def load_checkpoint(self, config, checkpoint_path, eval=False, use_cuda=False, criterion=None, cache=False):
        # pylint: disable=redefined-builtin,unused-argument
        """base_encoder.py:109-161 without the training criterion classes: a ``criterion`` passed in gets the
        checkpoint's criterion state."""
        state = torch.load(checkpoint_path, map_location=torch.device("cpu"), weights_only=False)
        try:
            self.load_state_dict(state["model"])
        except (KeyError, RuntimeError):
            if eval:
                raise
            own = self.state_dict()
            own.update({k: v for k, v in state["model"].items() if k in own and own[k].shape == v.shape})
            self.load_state_dict(own)
        if criterion is not None and "criterion" in state:
            try:
                criterion.load_state_dict(state["criterion"])
            except (KeyError, RuntimeError) as error:
                print(" > Criterion load ignored because of:", error)
        if use_cuda:
            self.cuda()
            if criterion is not None:
                criterion = criterion.cuda()
        if eval:
            self.eval()
        if not eval:
            return criterion, state["step"]
        return criterion


def setup_encoder_model(config):
    """generic_utils.py:118-136 for ``model_name == "resnet"``; the LSTM encoder is not built."""
    mp = config.model_params
    name = mp["model_name"].lower()
    if name == "lstm":
        raise NotImplementedError("tts_b200.setup_encoder_model: the LSTM speaker encoder is not built")
    if name != "resnet":
        raise ValueError(f"tts_b200.setup_encoder_model: unknown model_name {mp['model_name']!r}")
    return ResNetSpeakerEncoder(input_dim=mp["input_dim"], proj_dim=mp["proj_dim"], log_input=mp.get("log_input", False),
                                use_torch_spec=mp.get("use_torch_spec", False), audio_config=config.audio)
