"""Oracle for the Griffin-Lim chain: librosa's ``stft`` / ``istft`` (center=True, reflect padding, periodic Hann
window centred in n_fft, window-sum-square normalisation) restated in numpy, and the reference's inverse-spectrogram
chain (processor.py:444-458, numpy_transforms.py:220-230) on top of them.

``dtype`` selects the arithmetic of the Griffin-Lim loop: float64 / complex128 is the reference's; float32 / complex64
(scipy.fft keeps single precision) is the float32 yardstick the device result is measured against."""
import numpy as np
import scipy.fft
import scipy.signal


def hann(win_length, n_fft, dtype=np.float64):
    """scipy.signal.get_window("hann", win_length, fftbins=True) centred in n_fft (librosa's pad_center)."""
    w = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) / win_length)
    left = (n_fft - win_length) // 2
    return np.pad(w, (left, n_fft - win_length - left)).astype(dtype)


def stft(y, n_fft, hop_length, win_length, pad_mode="reflect"):
    """librosa.stft(y, n_fft, hop_length, win_length, window="hann", center=True, pad_mode) -> [F, T]."""
    w = hann(win_length, n_fft, y.dtype)
    yp = np.pad(y, n_fft // 2, mode=pad_mode)
    n_frames = 1 + (len(yp) - n_fft) // hop_length
    idx = np.arange(n_fft)[None, :] + hop_length * np.arange(n_frames)[:, None]
    return scipy.fft.rfft(yp[idx] * w[None, :], axis=-1).T


def istft(S, hop_length, win_length):
    """librosa.istft(S, hop_length, win_length, window="hann", center=True) -> hop (T - 1) samples."""
    n_fft = 2 * (S.shape[0] - 1)
    rdtype = np.float32 if S.dtype == np.complex64 else np.float64
    w = hann(win_length, n_fft, rdtype)
    frames = scipy.fft.irfft(S.T, n=n_fft, axis=-1) * w[None, :]
    n_frames = S.shape[1]
    n = n_fft + hop_length * (n_frames - 1)
    y = np.zeros(n, dtype=rdtype)
    wss = np.zeros(n, dtype=rdtype)
    for t in range(n_frames):
        y[t * hop_length: t * hop_length + n_fft] += frames[t]
        wss[t * hop_length: t * hop_length + n_fft] += w * w
    nz = wss > np.finfo(rdtype).tiny
    y[nz] /= wss[nz]
    return y[n_fft // 2: n - n_fft // 2]


def griffin_lim(spec, num_iter, hop_length, win_length, u, dtype=np.float64):
    """numpy_transforms.griffin_lim with the draws u (np.random.rand(*spec.shape)) given."""
    cdt = np.complex128 if dtype == np.float64 else np.complex64
    angles = np.exp(2j * np.pi * u.astype(np.float64)).astype(cdt)
    S = np.abs(spec).astype(cdt)
    y = istft(S * angles, hop_length, win_length)
    if not np.isfinite(y).all():
        return np.array([0.0])
    n_fft = 2 * (spec.shape[0] - 1)
    for _ in range(num_iter):
        angles = np.exp(1j * np.angle(stft(y, n_fft, hop_length, win_length))).astype(cdt)
        y = istft(S * angles, hop_length, win_length)
    return y


def denormalize(S, ap):
    """AudioProcessor.denormalize (processor.py:300-336) in float32; ap carries the constructor's fields, and
    ``stats`` = {"mel": (mean, std), "linear": (mean, std)} for the mean-var scaler."""
    S = S.copy()
    if not ap["signal_norm"]:
        return S
    if ap.get("stats") is not None:
        if S.shape[0] == ap["num_mels"]:
            mean, std = ap["stats"]["mel"]
        elif S.shape[0] == ap["fft_size"] / 2:
            mean, std = ap["stats"]["linear"]
        else:
            raise RuntimeError(" [!] Mean-Var stats does not match the given feature dimensions.")
        X = S.T.copy()                   # StandardScaler.inverse_transform: in place, so float32 stays float32
        X *= std
        X += mean
        return X.T
    mx, mn, ref = ap["max_norm"], ap["min_level_db"], ap["ref_level_db"]
    if ap["symmetric_norm"]:
        if ap["clip_norm"]:
            S = np.clip(S, -mx, mx)
        S = ((S + mx) * -mn / (2 * mx)) + mn
        return S + ref
    if ap["clip_norm"]:
        S = np.clip(S, 0, mx)
    S = (S * -mn / mx) + mn
    return S + ref


def magnitudes(S, ap, mel_basis=None):
    """|S| ** power of a normalised [C, T] spectrogram (float32, as the reference), mel through pinv(mel_basis)."""
    D = denormalize(S.astype(np.float32), ap)
    A = np.power(10, D / ap["spec_gain"]) if ap["base"] == 10 else np.exp(D / ap["spec_gain"])
    if mel_basis is not None:
        A = np.maximum(1e-10, np.dot(np.linalg.pinv(mel_basis), A))
    return A ** ap["power"]


def inv_spectrogram(S, ap, u, mel_basis=None, dtype=np.float64):
    """AudioProcessor.inv_spectrogram (mel_basis None) / inv_melspectrogram of one [C, T] row with draws u [F, T]."""
    W = griffin_lim(magnitudes(S, ap, mel_basis), ap["griffin_lim_iters"], ap["hop_length"], ap["win_length"], u, dtype)
    if ap["preemphasis"] != 0:
        W = scipy.signal.lfilter([1], [1, -ap["preemphasis"]], W)
    return W


def rel_rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(np.mean((a - b) ** 2)) / max(np.sqrt(np.mean(b ** 2)), 1e-30))


def spectral_convergence(y, S, n_fft, hop_length, win_length):
    """||  |STFT(y)| - S || / || S ||  (S the target magnitudes)."""
    X = np.abs(stft(np.asarray(y, np.float64), n_fft, hop_length, win_length))
    return float(np.linalg.norm(X - S) / np.linalg.norm(S))
