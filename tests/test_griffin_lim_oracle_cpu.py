"""The Griffin-Lim oracle (tests/griffin_lim_oracle.py) against torch's STFT and against the unmodified reference chain
(AudioProcessor.inv_spectrogram / inv_melspectrogram, numpy_transforms.griffin_lim, synthesis.apply_griffin_lim), and
the drop-in AudioProcessor's constructor surface."""
import numpy as np
import pytest
import torch

import griffin_lim_oracle as G
import ref_golden
from tts_b200.audio import AudioProcessor, mel_filterbank

GEOMETRIES = [(1024, 256, 1024), (2048, 275, 1102)]


@pytest.mark.parametrize("n_fft,hop,win", GEOMETRIES)
def test_oracle_stft_istft_match_torch(n_fft, hop, win):
    y = np.random.default_rng(0).standard_normal(9000)
    w = torch.from_numpy(G.hann(win, win))
    X = torch.stft(torch.from_numpy(y), n_fft, hop, win, window=w, center=True, pad_mode="reflect", return_complex=True)
    got = G.stft(y, n_fft, hop, win)
    assert got.shape == tuple(X.shape)
    assert np.abs(got - X.numpy()).max() <= 1e-12 * np.abs(got).max()
    yi = torch.istft(X, n_fft, hop, win, window=w, center=True).numpy()
    gi = G.istft(got, hop, win)
    assert gi.shape == (hop * (got.shape[1] - 1),)
    assert np.abs(gi - yi[: gi.shape[0]]).max() <= 1e-12 * np.abs(yi).max()


def test_oracle_stft_short_row_periodic_reflect():
    # 300 samples under a 1024-point frame: the reflect pad (512) exceeds the row, numpy's pad repeats the reflection
    y = np.random.default_rng(1).standard_normal(300)
    n_fft, hop, win = 1024, 256, 1024
    yp = np.pad(y, n_fft // 2, mode="reflect")
    frames = np.stack([yp[t * hop: t * hop + n_fft] * G.hann(win, n_fft) for t in range(1 + (len(yp) - n_fft) // hop)])
    want = np.fft.rfft(frames, axis=-1).T
    assert np.abs(G.stft(y, n_fft, hop, win) - want).max() <= 1e-12 * np.abs(want).max()


# --------------------------------------------------------------------------- against the unmodified reference
BASE_AP = dict(sample_rate=22050, num_mels=20, fft_size=256, hop_length=64, win_length=256, power=1.5,
               griffin_lim_iters=3, signal_norm=True, symmetric_norm=True, max_norm=4.0, clip_norm=True,
               min_level_db=-100, ref_level_db=20, spec_gain=20, log_func="np.log10", preemphasis=0.0)
CASES = {
    "symmetric_clip": {},
    "symmetric_noclip": dict(clip_norm=False),
    "asymmetric_clip": dict(symmetric_norm=False, max_norm=1.0),
    "asymmetric_noclip": dict(symmetric_norm=False, max_norm=1.0, clip_norm=False),
    "no_signal_norm": dict(signal_norm=False),
    "ln_gain1": dict(log_func="np.log", spec_gain=1),
    "preemphasis": dict(preemphasis=0.97),
    "stats": dict(stats=True),
    "win_lt_fft": dict(hop_length=55, win_length=220),
}


def oracle_ap(kw):
    ap = dict(BASE_AP, **kw)
    ap["base"] = np.e if ap["log_func"] == "np.log" else 10
    return ap


def inputs(kw, C, T, seed):
    g = np.random.default_rng(seed)
    if kw.get("signal_norm", True) is False:
        return (g.standard_normal((C, T)) * 10 - 20).astype(np.float32)
    if kw.get("stats"):
        return g.standard_normal((C, T)).astype(np.float32)
    lo = 0.0 if kw.get("symmetric_norm", True) is False else -4.0
    return (g.uniform(lo - 0.5, 4.5, (C, T))).astype(np.float32)


def stats_for(ap, tmp_path):
    g = np.random.default_rng(7)
    F = ap["fft_size"] // 2 + 1
    st = {"mel_mean": (g.standard_normal(ap["num_mels"]) * 5 - 30).astype(np.float32),
          "mel_std": (g.uniform(5, 10, ap["num_mels"])).astype(np.float32),
          "linear_mean": (g.standard_normal(F) * 5 - 30).astype(np.float32),
          "linear_std": (g.uniform(5, 10, F)).astype(np.float32),
          "audio_config": {"num_mels": ap["num_mels"], "fft_size": ap["fft_size"]}}
    path = tmp_path / "stats.npy"
    np.save(path, st, allow_pickle=True)
    return st, str(path)


def reference_ap(kw, tmp_path, monkeypatch):
    """The reference AudioProcessor with the oracle's stft / istft in librosa's place and the Slaney basis."""
    import ref_import

    mods = ref_import.load_full()
    import librosa  # the placeholder ref_import installs

    monkeypatch.setattr(librosa, "stft", lambda *, y, n_fft, hop_length, win_length, pad_mode, window, center:
                        G.stft(y, n_fft, hop_length, win_length, pad_mode), raising=False)
    monkeypatch.setattr(librosa, "istft", lambda y, *, hop_length, win_length, center, window:
                        G.istft(y, hop_length, win_length), raising=False)
    args = {k: v for k, v in dict(BASE_AP, **kw).items() if k != "stats"}
    st = None
    if kw.get("stats"):
        st, args["stats_path"] = stats_for(dict(BASE_AP, **kw), tmp_path)
    ap = mods["processor"].AudioProcessor(verbose=False, **args)
    ap.mel_basis = mel_filterbank(args["sample_rate"], args["fft_size"], args["num_mels"], ap.mel_fmin, ap.mel_fmax)
    return mods, ap, st


def oracle_run(kw, S, mel, tmp_path, seed, stats=None):
    ap = oracle_ap(kw)
    if kw.get("stats"):
        st = stats if stats is not None else stats_for(ap, tmp_path)[0]
        ap["stats"] = {"mel": (st["mel_mean"], st["mel_std"]), "linear": (st["linear_mean"], st["linear_std"])}
    basis = mel_filterbank(ap["sample_rate"], ap["fft_size"], ap["num_mels"]) if mel else None
    np.random.seed(seed)
    u = np.random.rand(ap["fft_size"] // 2 + 1, S.shape[1])
    return G.inv_spectrogram(S, ap, u, basis)


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("mel", [True, False], ids=["mel", "linear"])
def test_oracle_equals_reference(case, mel, tmp_path, monkeypatch):
    kw = CASES[case]
    name = f"test_griffin_lim_oracle_equals_reference[{case}-{'mel' if mel else 'linear'}]"
    rec = ref_golden.Recorded(name)
    C = BASE_AP["num_mels"] if mel else BASE_AP["fft_size"] // 2 + 1
    S = inputs(kw, C, 12, seed=3)
    if kw.get("stats") and not mel:
        # the linear scaler only takes fft_size / 2 channels: a full linear spectrogram raises
        def ref_err():
            mods, ap, _ = reference_ap(kw, tmp_path, monkeypatch)
            try:
                ap.inv_spectrogram(S)
            except RuntimeError as e:
                return str(e)
            return None
        msg = rec.value("error", ref_err)
        assert msg is not None and "Mean-Var" in msg
        with pytest.raises(RuntimeError, match="Mean-Var"):
            oracle_run(kw, S, mel, tmp_path, 5)
        rec.save()
        return

    def ref():
        mods, ap, _ = reference_ap(kw, tmp_path, monkeypatch)
        np.random.seed(5)
        return torch.from_numpy(np.asarray(ap.inv_melspectrogram(S) if mel else ap.inv_spectrogram(S)))

    got = torch.from_numpy(np.asarray(oracle_run(kw, S, mel, tmp_path, 5)))
    rec.check("wav", got, ref)
    rec.save()


def test_oracle_griffin_lim_and_non_finite_equal_reference(tmp_path, monkeypatch):
    rec = ref_golden.Recorded("test_oracle_griffin_lim_and_non_finite_equal_reference")
    g = np.random.default_rng(4)
    spec = g.uniform(0, 2, (129, 10))
    bad = spec.copy()
    bad[3, 4] = np.inf

    def ref(x):
        mods, _, _ = reference_ap({}, tmp_path, monkeypatch)
        np.random.seed(9)
        return torch.from_numpy(np.asarray(mods["numpy_transforms"].griffin_lim(
            spec=x, num_iter=4, hop_length=64, win_length=256, fft_size=256, pad_mode="reflect"), dtype=np.float64))

    np.random.seed(9)
    got = G.griffin_lim(spec, 4, 64, 256, np.random.rand(*spec.shape))
    rec.check("finite", torch.from_numpy(got), lambda: ref(spec))
    np.random.seed(9)
    got_bad = G.griffin_lim(bad, 4, 64, 256, np.random.rand(*bad.shape))
    assert np.array_equal(got_bad, np.array([0.0]))
    rec.check("non_finite", torch.from_numpy(got_bad), lambda: ref(bad))
    rec.save()


def test_oracle_apply_griffin_lim_equals_reference(tmp_path, monkeypatch):
    rec = ref_golden.Recorded("test_oracle_apply_griffin_lim_equals_reference")
    kw = CASES["symmetric_clip"]
    g = np.random.default_rng(6)
    x = g.uniform(-4, 4, (3, 14, BASE_AP["num_mels"])).astype(np.float32)   # [B, T, C], full padded rows
    lens = np.array([14, 9, 5])

    def ref():
        mods, ap, _ = reference_ap(kw, tmp_path, monkeypatch)

        class Cfg:
            model = "glow_tts"
        np.random.seed(11)
        wavs = mods["synthesis"].apply_griffin_lim(x, lens, Cfg, ap)
        return torch.from_numpy(np.concatenate(wavs))

    ap = oracle_ap(kw)
    basis = mel_filterbank(ap["sample_rate"], ap["fft_size"], ap["num_mels"])
    np.random.seed(11)
    wavs = []
    for b in range(3):
        u = np.random.rand(ap["fft_size"] // 2 + 1, x.shape[1])
        w = G.inv_spectrogram(x[b].T, ap, u, basis)
        wavs.append(w[: lens[b] * ap["hop_length"] - ap["hop_length"]])
    rec.check("wavs", torch.from_numpy(np.concatenate(wavs)), ref)
    rec.check("lengths", torch.tensor([len(w) for w in wavs]), lambda: torch.tensor([len(w) for w in wavs]))
    rec.save()


SURFACE = {
    "defaults": dict(sample_rate=22050, num_mels=80, hop_length=256, win_length=1024),
    "ms_derived": dict(sample_rate=22050, num_mels=80, frame_shift_ms=12.5, frame_length_ms=50, fft_size=2048,
                       power=1.5, griffin_lim_iters=60, preemphasis=0.97, signal_norm=True, symmetric_norm=True,
                       max_norm=4.0, min_level_db=-100, ref_level_db=20, mel_fmax=8000.0, unrelated_key=3),
}
FIELDS = ["sample_rate", "num_mels", "log_func", "min_level_db", "ref_level_db", "fft_size", "power", "preemphasis",
          "griffin_lim_iters", "signal_norm", "symmetric_norm", "mel_fmin", "mel_fmax", "spec_gain", "stft_pad_mode",
          "max_norm", "clip_norm", "hop_length", "win_length", "base", "stats_path"]


@pytest.mark.parametrize("case", sorted(SURFACE))
def test_audio_processor_surface_matches_reference(case):
    rec = ref_golden.Recorded(f"test_audio_processor_surface_matches_reference[{case}]")

    def ref():
        import ref_import

        mods = ref_import.load_full()
        ap = mods["processor"].AudioProcessor(verbose=False, **SURFACE[case])
        return {k: (float(v) if isinstance(v, (float, np.floating)) else v) for k, v in
                ((k, getattr(ap, k)) for k in FIELDS)}

    want = rec.value("fields", ref)
    ap = AudioProcessor(verbose=False, **SURFACE[case])
    got = {k: (float(v) if isinstance(v, (float, np.floating)) else v) for k, v in ((k, getattr(ap, k)) for k in FIELDS)}
    assert got == want
    rec.save()
