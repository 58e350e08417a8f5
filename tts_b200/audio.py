"""Drop-ins for the STFT / mel front end on the hot path:
``wav_to_spec`` / ``spec_to_mel`` / ``wav_to_mel`` / ``amp_to_db`` / ``db_to_amp``
(/root/reference/TTS/tts/models/vits.py:78-208) and ``TorchSTFT``
(/root/reference/TTS/utils/audio/torch_transforms.py:6-165), computed by libtts_b200.so.

The mel filterbank is the Slaney-style ``librosa.filters.mel`` (htk=False, norm="slaney") the reference
calls; librosa is not a dependency here, ``mel_filterbank`` below builds the same matrix on the host.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib

_handles = {}


def mel_filterbank(sample_rate, n_fft, n_mels, fmin=0.0, fmax=None):
    """Triangular mel filters on the Slaney scale (linear below 1 kHz, log above), area-normalised."""
    fmax = float(sample_rate) / 2.0 if fmax is None else float(fmax)
    lin_step, knee_hz = 200.0 / 3.0, 1000.0
    knee_mel, log_step = knee_hz / lin_step, math.log(6.4) / 27.0

    def to_mel(hz):
        hz = np.asarray(hz, dtype=np.float64)
        return np.where(hz >= knee_hz, knee_mel + np.log(np.maximum(hz, 1e-10) / knee_hz) / log_step, hz / lin_step)

    def to_hz(mel):
        mel = np.asarray(mel, dtype=np.float64)
        return np.where(mel >= knee_mel, knee_hz * np.exp(log_step * (mel - knee_mel)), mel * lin_step)

    edges = to_hz(np.linspace(to_mel(fmin), to_mel(fmax), n_mels + 2))
    bins = np.fft.rfftfreq(n_fft, d=1.0 / sample_rate)
    width = np.diff(edges)
    rel = edges[:, None] - bins[None, :]
    fb = np.zeros((n_mels, bins.shape[0]), dtype=np.float32)
    for m in range(n_mels):
        rising = -rel[m] / width[m]
        falling = rel[m + 2] / width[m + 1]
        fb[m] = np.maximum(0.0, np.minimum(rising, falling))
    fb *= (2.0 / (edges[2:] - edges[:-2]))[:, None]
    return fb


def _window(win_length, n_fft, name="hann_window"):
    w = getattr(torch, name)(win_length).to(torch.float32)
    if win_length < n_fft:  # torch.stft centres a short window inside the frame
        left = (n_fft - win_length) // 2
        w = torch.nn.functional.pad(w, (left, n_fft - win_length - left))
    return w.contiguous()


def _handle(device, n_fft, hop, win_length, window_name, mel_key=None, mel_basis=None):
    key = (str(device), n_fft, hop, win_length, window_name, mel_key)
    h = _handles.get(key)
    if h is None:
        w = _window(win_length, n_fft, window_name)
        mb = None if mel_basis is None else torch.as_tensor(mel_basis, dtype=torch.float32).contiguous()
        out = ctypes.c_void_p()
        with torch.cuda.device(device):
            rc = _lib.lib().b200tts_stft_create(n_fft, hop, _lib.ptr(w), _lib.ptr(mb),
                                                0 if mb is None else mb.shape[0], ctypes.byref(out))
        _lib.check(rc, "stft_create")
        _handles[key] = h = out
    return h


def _magnitude(h, y, n_fft, hop, pad1, pad2, mode, power=1.0):
    _lib.require_cuda(y, "y")
    y = y.to(torch.float32).contiguous()
    b, t = y.shape
    n_frames = 1 + (t + 2 * pad1 + 2 * pad2 - n_fft) // hop
    spec = torch.empty((b, n_fft // 2 + 1, max(n_frames, 0)), dtype=torch.float32, device=y.device)
    with torch.cuda.device(y.device):
        rc = _lib.lib().b200tts_stft_magnitude(h, _lib.ptr(y), b, t, pad1, pad2, mode, ctypes.c_float(power),
                                               _lib.ptr(spec), n_frames, _lib.stream_ptr(y.device))
    _lib.check(rc, "stft_magnitude")
    return spec


def _project(h, spec, n_mels, log_clamp):
    spec = spec.contiguous()
    b, _, n = spec.shape
    mel = torch.empty((b, n_mels, n), dtype=torch.float32, device=spec.device)
    with torch.cuda.device(spec.device):
        rc = _lib.lib().b200tts_stft_mel_project(h, _lib.ptr(spec), b, n, ctypes.c_float(log_clamp), _lib.ptr(mel),
                                                 _lib.stream_ptr(spec.device))
    _lib.check(rc, "stft_mel_project")
    return mel


def amp_to_db(magnitudes, C=1, clip_val=1e-5):
    return torch.log(torch.clamp(magnitudes, min=clip_val) * C)


def db_to_amp(magnitudes, C=1):
    return torch.exp(magnitudes) / C


def wav_to_spec(y, n_fft, hop_length, win_length, center=False):
    """y [B,1,T] -> linear magnitude spectrogram [B, n_fft/2+1, frames]   (vits.py:96-138)."""
    if center:
        raise NotImplementedError("tts_b200.wav_to_spec: the reference only calls this with center=False")
    y = y.squeeze(1)
    h = _handle(y.device, n_fft, hop_length, win_length, "hann_window")
    return _magnitude(h, y, n_fft, hop_length, int((n_fft - hop_length) / 2), 0, mode=0)


def spec_to_mel(spec, n_fft, num_mels, sample_rate, fmin, fmax):
    """[B, n_fft/2+1, T] -> log-mel [B, num_mels, T]   (vits.py:141-157)."""
    _lib.require_cuda(spec, "spec")
    basis = mel_filterbank(sample_rate, n_fft, num_mels, fmin, fmax)
    h = _handle(spec.device, n_fft, 1, n_fft, "hann_window", mel_key=(sample_rate, num_mels, fmin, fmax), mel_basis=basis)
    return _project(h, spec.to(torch.float32), num_mels, 1e-5)


def wav_to_mel(y, n_fft, num_mels, sample_rate, hop_length, win_length, fmin, fmax, center=False):
    """y [B,1,T] -> log-mel [B, num_mels, frames]   (vits.py:160-208)."""
    return spec_to_mel(wav_to_spec(y, n_fft, hop_length, win_length, center), n_fft, num_mels, sample_rate, fmin, fmax)


class TorchSTFT(torch.nn.Module):
    """Same constructor and call contract as TTS.utils.audio.torch_transforms.TorchSTFT."""

    def __init__(self, n_fft, hop_length, win_length, pad_wav=False, window="hann_window", sample_rate=None,
                 mel_fmin=0, mel_fmax=None, n_mels=80, use_mel=False, do_amp_to_db=False, spec_gain=1.0, power=None,
                 use_htk=False, mel_norm="slaney", normalized=False):
        super().__init__()
        if use_htk or mel_norm != "slaney" or normalized:
            raise NotImplementedError("tts_b200.TorchSTFT: only the Slaney mel / un-normalised STFT is built")
        self.n_fft, self.hop_length, self.win_length, self.pad_wav = n_fft, hop_length, win_length, pad_wav
        self.sample_rate, self.mel_fmin, self.mel_fmax, self.n_mels = sample_rate, mel_fmin, mel_fmax, n_mels
        self.use_mel, self.do_amp_to_db, self.spec_gain, self.power = use_mel, do_amp_to_db, spec_gain, power
        self.window_name = window
        self.window = torch.nn.Parameter(getattr(torch, window)(win_length), requires_grad=False)
        self.mel_basis = None
        if use_mel:
            self.mel_basis = torch.from_numpy(mel_filterbank(sample_rate, n_fft, n_mels, mel_fmin, mel_fmax)).float()

    def __call__(self, x):
        """x [B,T] or [B,1,T] -> [B, n_fft/2+1 or n_mels, frames]   (torch_transforms.py:104-145)."""
        if x.ndim == 3:
            x = x.squeeze(1)
        key = (self.sample_rate, self.n_mels, self.mel_fmin, self.mel_fmax) if self.use_mel else None
        h = _handle(x.device, self.n_fft, self.hop_length, self.win_length, self.window_name, mel_key=key,
                    mel_basis=None if self.mel_basis is None else self.mel_basis.numpy())
        pad1 = int((self.n_fft - self.hop_length) / 2) if self.pad_wav else 0
        s = _magnitude(h, x, self.n_fft, self.hop_length, pad1, self.n_fft // 2, mode=1,
                       power=1.0 if self.power is None else float(self.power))
        if self.use_mel:
            s = _project(h, s, self.n_mels, 0.0)
        if self.do_amp_to_db:
            s = torch.log(torch.clamp(s, min=1e-5) * self.spec_gain)
        return s


# ----------------------------------------------------------------------------- Griffin-Lim (TTS/utils/audio mirror)
def millisec_to_length(*, frame_length_ms=None, frame_shift_ms=None, sample_rate=None, **kwargs):
    """(win_length, hop_length) from milliseconds, as numpy_transforms.millisec_to_length."""
    factor = frame_length_ms / frame_shift_ms
    assert (factor).is_integer(), " [!] frame_shift_ms should divide frame_length_ms"
    win_length = int(frame_length_ms / 1000.0 * sample_rate)
    hop_length = int(win_length / float(factor))
    return win_length, hop_length


def _norm_c(signal_norm, symmetric_norm, clip_norm, max_norm, min_level_db, ref_level_db, mean=None, std=None):
    s = _lib.AudioNormC()
    s.signal_norm, s.symmetric_norm, s.clip_norm = int(bool(signal_norm)), int(bool(symmetric_norm)), int(bool(clip_norm))
    s.max_norm = float(max_norm or 0.0)
    s.min_level_db, s.ref_level_db = float(min_level_db or 0.0), float(ref_level_db or 0.0)
    if mean is not None:
        s.scaler_mean, s.scaler_scale = mean.data_ptr(), std.data_ptr()
    return s


class _GlHandle:
    """One b200tts_griffin_lim handle (window, twiddles, optional pinv(mel_basis) on the device), destroyed with its
    owner."""

    def __init__(self, device, n_fft, hop, win_length, pinv=None):
        self.h = None
        w = _window(win_length, n_fft)
        p = None if pinv is None else torch.from_numpy(np.ascontiguousarray(pinv, dtype=np.float32))
        out = ctypes.c_void_p()
        with torch.cuda.device(device):
            rc = _lib.lib().b200tts_griffin_lim_create(n_fft, hop, _lib.ptr(w), _lib.ptr(p),
                                                       0 if p is None else p.shape[1], ctypes.byref(out))
        _lib.check(rc, "griffin_lim_create")
        self.h = out

    def __del__(self):
        if self.h is not None:
            try:
                _lib.lib().b200tts_griffin_lim_destroy(self.h)
            except Exception:   # noqa: BLE001 -- interpreter shutdown: the process frees the device anyway
                pass
            self.h = None


_gl_linear = {}   # linear handles hold only the window and twiddles: one per (device, geometry)


def _gl_linear_handle(device, n_fft, hop, win_length):
    key = (str(device), n_fft, hop, win_length)
    h = _gl_linear.get(key)
    if h is None:
        _gl_linear[key] = h = _GlHandle(device, n_fft, hop, win_length)
    return h


def _check_geometry(fft_size, hop_length, win_length, pad_mode):
    if pad_mode != "reflect":
        raise NotImplementedError(f"tts_b200: Griffin-Lim is built for stft_pad_mode='reflect' only, got {pad_mode!r}")
    if fft_size < 32 or fft_size > 8192 or fft_size & (fft_size - 1):
        raise NotImplementedError(f"tts_b200: Griffin-Lim needs a power-of-two fft_size in [32, 8192], got {fft_size}")
    if not 1 <= win_length <= fft_size or not 1 <= hop_length <= win_length:
        raise ValueError(f"tts_b200: Griffin-Lim needs 1 <= hop_length ({hop_length}) <= win_length ({win_length}) "
                         f"<= fft_size ({fft_size})")


def _griffin_lim_call(x, C, handle, *, fft_size, hop_length, win_length, pad_mode, num_iter, norm_c, base, spec_gain,
                      power, preemphasis, lengths=None, angles=None, time_last=True):
    """The batched device chain on x: [C, T] / [B, C, T] (``time_last``) or [T, C] / [B, T, C].  ``handle`` is a callable
    giving the _GlHandle for a device.  Returns (wav [B, pitch], wav_lengths [B] int32, squeeze) with squeeze True for
    2-D input."""
    _check_geometry(fft_size, hop_length, win_length, pad_mode)
    _lib.require_cuda(x, "spectrogram")
    squeeze = x.dim() == 2
    if squeeze:
        if lengths is not None:
            raise ValueError("tts_b200: lengths= goes with batched [B, C, T] / [B, T, C] input")
        x = x.unsqueeze(0)
    if x.dim() != 3:
        raise ValueError(f"tts_b200: expected a [C, T] or batched spectrogram, got shape {tuple(x.shape)}")
    x = x.to(torch.float32)
    if time_last:                         # [B, C, T]
        b, c, t = x.shape
        sb, sc, st = x.stride()
    else:                                 # [B, T, C], e.g. a TTS model's output
        b, t, c = x.shape
        sb, st, sc = x.stride()
    if c != C:
        layout = "[B, C, T]" if time_last else "[B, T, C]"
        raise ValueError(f"tts_b200: expected {C} channels on the channel axis of a {layout} spectrogram "
                         f"(time_last={time_last}), got shape {tuple(x.shape)}")
    F = fft_size // 2 + 1
    dev = x.device
    lens_host = [t] * b if lengths is None else [int(v) for v in torch.as_tensor(lengths).reshape(-1).tolist()]
    if len(lens_host) != b or any(v > t for v in lens_host):
        raise ValueError(f"tts_b200: lengths must hold {b} frame counts <= {t}, got {lens_host}")
    if min(lens_host) < 2:
        raise ValueError("tts_b200: Griffin-Lim needs at least 2 frames per row (1 frame gives an empty waveform)")
    if angles is None:                    # numpy's global RNG, row by row, as the reference draws them
        u = np.zeros((b, F, t), dtype=np.float32)
        for i, tb in enumerate(lens_host):
            u[i, :, :tb] = np.random.rand(F, tb)
        u = torch.from_numpy(u).to(dev)
    else:
        u = torch.as_tensor(angles).to(dev, torch.float32)
        u = u.unsqueeze(0) if u.dim() == 2 else u
        if u.shape[0] != b or u.shape[1] != F or u.shape[2] < max(lens_host):
            raise ValueError(f"tts_b200: angles must be [{b}, {F}, >= {max(lens_host)}], got {tuple(u.shape)}")
        if u.shape[2] != t:
            u = torch.nn.functional.pad(u[:, :, :t], (0, max(0, t - u.shape[2])))
        u = u.contiguous()
    lens_d = None if lengths is None else torch.tensor(lens_host, dtype=torch.int32, device=dev)
    h = handle(dev).h
    L = hop_length * (t - 1)
    wav = torch.empty((b, L), dtype=torch.float32, device=dev)
    wav_lengths = torch.empty((b,), dtype=torch.int32, device=dev)
    L_ = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = L_.b200tts_griffin_lim_workspace_bytes(h, b, t)
        ws = _lib.workspace(dev, nbytes, "griffin_lim")
        rc = L_.b200tts_griffin_lim_forward(h, _lib.ptr(x), sb, sc, st, b, C, t, _lib.ptr(lens_d), ctypes.byref(norm_c),
                                            float(base), float(spec_gain), float(power), int(num_iter),
                                            float(preemphasis), _lib.ptr(u), _lib.ptr(wav), L, _lib.ptr(wav_lengths),
                                            _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
    _lib.check(rc, "griffin_lim_forward")
    return wav, wav_lengths, squeeze


def griffin_lim(*, spec=None, num_iter=60, hop_length=None, win_length=None, fft_size=None, pad_mode="reflect",
                angles=None, lengths=None, time_last=True, **kwargs):
    """``numpy_transforms.griffin_lim`` on a CUDA magnitude spectrogram [F, T] (or batched [B, F, T] with ``lengths=``;
    ``time_last=False`` for [T, F] / [B, T, F]).  ``angles`` are the uniform draws u of ``np.random.rand(*spec.shape)``;
    without them numpy's global RNG draws them."""
    win_length = fft_size if win_length is None else win_length
    hop_length = win_length // 4 if hop_length is None else hop_length
    wav, wav_lengths, squeeze = _griffin_lim_call(
        spec, fft_size // 2 + 1, lambda dev: _gl_linear_handle(dev, fft_size, hop_length, win_length),
        fft_size=fft_size, hop_length=hop_length, win_length=win_length, pad_mode=pad_mode, num_iter=num_iter,
        norm_c=_norm_c(False, False, False, 0, 0, 0), base=0.0, spec_gain=1.0, power=1.0, preemphasis=0.0,
        lengths=lengths, angles=angles, time_last=time_last)
    return _finish(wav, wav_lengths, squeeze)


def _finish(wav, wav_lengths, squeeze):
    if squeeze:     # one row: trim to its length (1 sample for a non-finite row), a host read of one int
        return wav[0, : int(wav_lengths[0])]
    return wav, wav_lengths


class AudioProcessor:
    """The inverse-spectrogram half of ``TTS.utils.audio.AudioProcessor`` (processor.py:141-484) on the device:
    ``denormalize``, ``inv_spectrogram``, ``inv_melspectrogram`` with Griffin-Lim.  Same constructor keywords
    (unrelated ones are accepted and ignored, as the reference's ``**_``) and ``init_from_config``.

    The methods take a CUDA [C, T] spectrogram like the reference and return the waveform; or a batch [B, C, T] with
    ``lengths=`` (frames per row, default all) and return ``(wav [B, hop (T - 1)], wav_lengths [B])``, each row zero
    past its length.  ``time_last=False`` takes [T, C] / [B, T, C] instead (a TTS model's output): the layout is never
    guessed from the shape.  The spectrogram stays on the device; ``lengths`` (B frame counts) is read to the host,
    where it is checked and sizes the default phase draws.  ``angles=`` gives the phase draws u in [0, 1) as [B, F, T] (F = fft_size / 2 + 1);
    without it the host draws ``np.random.rand(F, T_b)`` row by row, so ``np.random.seed(s)`` reproduces the
    reference's draws."""

    def __init__(self, sample_rate=None, resample=False, num_mels=None, log_func="np.log10", min_level_db=None,
                 frame_shift_ms=None, frame_length_ms=None, hop_length=None, win_length=None, ref_level_db=None,
                 fft_size=1024, power=None, preemphasis=0.0, signal_norm=None, symmetric_norm=None, max_norm=None,
                 mel_fmin=None, mel_fmax=None, pitch_fmax=None, pitch_fmin=None, spec_gain=20, stft_pad_mode="reflect",
                 clip_norm=True, griffin_lim_iters=None, do_trim_silence=False, trim_db=60, do_sound_norm=False,
                 do_amp_to_db_linear=True, do_amp_to_db_mel=True, do_rms_norm=False, db_level=None, stats_path=None,
                 verbose=True, **_):
        self.sample_rate = sample_rate
        self.resample = resample
        self.num_mels = num_mels
        self.log_func = log_func
        self.min_level_db = min_level_db or 0
        self.frame_shift_ms = frame_shift_ms
        self.frame_length_ms = frame_length_ms
        self.ref_level_db = ref_level_db
        self.fft_size = fft_size
        self.power = power
        self.preemphasis = preemphasis
        self.griffin_lim_iters = griffin_lim_iters
        self.signal_norm = signal_norm
        self.symmetric_norm = symmetric_norm
        self.mel_fmin = mel_fmin or 0
        self.mel_fmax = mel_fmax
        self.pitch_fmin = pitch_fmin
        self.pitch_fmax = pitch_fmax
        self.spec_gain = float(spec_gain)
        self.stft_pad_mode = stft_pad_mode
        self.max_norm = 1.0 if max_norm is None else float(max_norm)
        self.clip_norm = clip_norm
        self.do_trim_silence = do_trim_silence
        self.trim_db = trim_db
        self.do_sound_norm = do_sound_norm
        self.do_amp_to_db_linear = do_amp_to_db_linear
        self.do_amp_to_db_mel = do_amp_to_db_mel
        self.do_rms_norm = do_rms_norm
        self.db_level = db_level
        self.stats_path = stats_path
        if log_func == "np.log":
            self.base = np.e
        elif log_func == "np.log10":
            self.base = 10
        else:
            raise ValueError(" [!] unknown `log_func` value.")
        if hop_length is None:
            self.win_length, self.hop_length = millisec_to_length(
                frame_length_ms=self.frame_length_ms, frame_shift_ms=self.frame_shift_ms, sample_rate=self.sample_rate)
        else:
            self.hop_length = hop_length
            self.win_length = win_length
        assert min_level_db != 0.0, " [!] min_level_db is 0"
        assert self.win_length <= self.fft_size, \
            f" [!] win_length cannot be larger than fft_size - {self.win_length} vs {self.fft_size}"
        self.mel_basis = None
        if sample_rate is not None and num_mels is not None:
            if mel_fmax is not None:
                assert mel_fmax <= sample_rate // 2
                assert mel_fmax - self.mel_fmin > 0
            self.mel_basis = mel_filterbank(sample_rate, fft_size, num_mels, self.mel_fmin, mel_fmax)
        self._stats = None
        self._pinv_of, self._pinv, self._mel_handles = None, None, {}
        if stats_path and signal_norm:
            mel_mean, mel_std, linear_mean, linear_std, _ = self.load_stats(stats_path)
            self.setup_scaler(mel_mean, mel_std, linear_mean, linear_std)
            self.signal_norm = True
            self.max_norm = None
            self.clip_norm = None
            self.symmetric_norm = None

    @staticmethod
    def init_from_config(config, verbose=True):
        if "audio" in config:
            return AudioProcessor(verbose=verbose, **config.audio)
        return AudioProcessor(verbose=verbose, **config)

    def load_stats(self, stats_path):
        """(mel_mean, mel_std, linear_mean, linear_std, audio_config) of a stats ``.npy``, with the reference's checks
        that the statistics were computed with this processor's settings."""
        stats = np.load(stats_path, allow_pickle=True).item()
        stats_config = stats["audio_config"]
        skip_parameters = ["griffin_lim_iters", "stats_path", "do_trim_silence", "ref_level_db", "power"]
        for key in stats_config.keys():
            if key in skip_parameters:
                continue
            if key not in ["sample_rate", "trim_db"]:
                assert stats_config[key] == self.__dict__[key], \
                    f" [!] Audio param {key} does not match the value used for computing mean-var stats. " \
                    f"{stats_config[key]} vs {self.__dict__[key]}"
        return stats["mel_mean"], stats["mel_std"], stats["linear_mean"], stats["linear_std"], stats_config

    def setup_scaler(self, mel_mean, mel_std, linear_mean, linear_std):
        self._stats = {"mel": (np.asarray(mel_mean), np.asarray(mel_std)),
                       "linear": (np.asarray(linear_mean), np.asarray(linear_std))}

    # ------------------------------------------------------------------ device chain
    def _norm(self, C, device, keep):
        """The b200tts_audio_norm of ``denormalize`` for a C-channel spectrogram (the mean-var scaler by channel count:
        num_mels -> mel, fft_size / 2 -> linear, anything else a RuntimeError, as the reference)."""
        if self._stats is None or not self.signal_norm:
            return _norm_c(self.signal_norm, self.symmetric_norm, self.clip_norm, self.max_norm, self.min_level_db,
                           self.ref_level_db)
        if C == self.num_mels:
            mean, std = self._stats["mel"]
        elif C == self.fft_size / 2:
            mean, std = self._stats["linear"]
        else:
            raise RuntimeError(" [!] Mean-Var stats does not match the given feature dimensions.")
        m = torch.as_tensor(mean, dtype=torch.float32).to(device).contiguous()
        s = torch.as_tensor(std, dtype=torch.float32).to(device).contiguous()
        keep += [m, s]
        return _norm_c(True, False, False, 0, 0, 0, m, s)

    def _mel_handle(self, device):
        """The mel handle of this processor on `device`: pinv(mel_basis) (np.linalg.pinv of the float32 basis, as
        mel_to_spec) computed once per basis, uploaded once per device."""
        if self._pinv_of is not self.mel_basis:
            self._pinv_of, self._pinv, self._mel_handles = self.mel_basis, np.linalg.pinv(self.mel_basis), {}
        key = str(device)
        h = self._mel_handles.get(key)
        if h is None:
            self._mel_handles[key] = h = _GlHandle(device, self.fft_size, self.hop_length, self.win_length, self._pinv)
        return h

    def _run(self, x, mel, lengths, angles, time_last):
        if self.power is None:
            raise ValueError("tts_b200: AudioProcessor.power is None; the reference raises on S ** None")
        _lib.require_cuda(x, "spectrogram")
        F = self.fft_size // 2 + 1
        C = self.num_mels if mel else F
        if mel:
            if self.mel_basis is None:
                raise ValueError("tts_b200: inv_melspectrogram needs sample_rate and num_mels")
            handle = self._mel_handle
        else:
            handle = lambda dev: _gl_linear_handle(dev, self.fft_size, self.hop_length, self.win_length)  # noqa: E731
        keep = []
        # the linear scaler only matches fft_size / 2 channels, which a linear spectrogram never has: raise before work
        norm = self._norm(C, x.device, keep)
        wav, wav_lengths, squeeze = _griffin_lim_call(
            x, C, handle, fft_size=self.fft_size, hop_length=self.hop_length, win_length=self.win_length,
            pad_mode=self.stft_pad_mode, num_iter=self.griffin_lim_iters, norm_c=norm, base=float(self.base),
            spec_gain=self.spec_gain, power=self.power, preemphasis=self.preemphasis, lengths=lengths, angles=angles,
            time_last=time_last)
        return _finish(wav, wav_lengths, squeeze)

    def denormalize(self, S):
        """``AudioProcessor.denormalize`` of a CUDA [C, T] / [B, C, T] spectrogram."""
        from .vocoder import AudioNorm, vocoder_input

        _lib.require_cuda(S, "S")
        C = S.shape[-2]
        if self._stats is not None and self.signal_norm:
            if C == self.num_mels:
                mean, std = self._stats["mel"]
            elif C == self.fft_size / 2:
                mean, std = self._stats["linear"]
            else:
                raise RuntimeError(" [!] Mean-Var stats does not match the given feature dimensions.")
            norm = AudioNorm(signal_norm=True, mel_mean=torch.as_tensor(mean), mel_std=torch.as_tensor(std))
        else:
            norm = AudioNorm(signal_norm=bool(self.signal_norm), symmetric_norm=bool(self.symmetric_norm),
                             max_norm=self.max_norm, clip_norm=bool(self.clip_norm), min_level_db=self.min_level_db,
                             ref_level_db=self.ref_level_db or 0.0)
        return vocoder_input(S, norm, AudioNorm.identity())

    def inv_spectrogram(self, spectrogram, *, lengths=None, angles=None, time_last=True):
        """``AudioProcessor.inv_spectrogram``: a normalised linear spectrogram -> waveform (Griffin-Lim)."""
        return self._run(spectrogram, False, lengths, angles, time_last)

    def inv_melspectrogram(self, mel_spectrogram, *, lengths=None, angles=None, time_last=True):
        """``AudioProcessor.inv_melspectrogram``: a normalised mel spectrogram -> waveform (Griffin-Lim)."""
        return self._run(mel_spectrogram, True, lengths, angles, time_last)


def inv_spectrogram(postnet_output, ap, CONFIG, *, angles=None):
    """``synthesis.inv_spectrogram``: postnet_output [T, C] -> waveform; linear for ``CONFIG.model == "tacotron"``."""
    if CONFIG.model.lower() in ["tacotron"]:
        return ap.inv_spectrogram(postnet_output.T, angles=angles)
    return ap.inv_melspectrogram(postnet_output.T, angles=angles)


def apply_griffin_lim(inputs, input_lens, CONFIG, ap, *, angles=None):
    """``synthesis.apply_griffin_lim``: every row of inputs [B, T, C] on its full padded spectrogram, in one batched
    device call, then trimmed to ``input_lens[b] * hop_length - hop_length`` samples.  Returns a list of CUDA tensors."""
    if CONFIG.model.lower() in ["tacotron"]:
        wav, wav_lengths = ap.inv_spectrogram(inputs, angles=angles, time_last=False)
    else:
        wav, wav_lengths = ap.inv_melspectrogram(inputs, angles=angles, time_last=False)
    have = wav_lengths.tolist()
    wavs = []
    for idx, n in enumerate(torch.as_tensor(input_lens).reshape(-1).tolist()):
        row = wav[idx, : have[idx]]
        wavs.append(row[: int(n) * ap.hop_length - ap.hop_length])
    return wavs
