"""Griffin-Lim on the GPU against the float64 oracle (tests/griffin_lim_oracle.py): the first iterations, 60 iterations
on harmonic-plus-noise speech-like signals for both STFT geometries and both input kinds, every case of the CPU suite,
a ragged 33-row batch against single-row calls and apply_griffin_lim, numpy's default draws, a non-finite row,
repeatability over a NaN-poisoned workspace with the launch list, both layouts when the frame count equals the channel
count, the Tacotron linear and Glow-TTS mel chains, and the rejected inputs."""
import numpy as np
import pytest
import scipy.signal
import torch

import griffin_lim_oracle as G
from test_griffin_lim_oracle_cpu import BASE_AP, CASES, inputs, oracle_ap, stats_for
from tts_b200 import _lib
from tts_b200.audio import AudioProcessor, apply_griffin_lim, griffin_lim, mel_filterbank

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SR = 22050
GEOM = {"1024/256/1024": (1024, 256, 1024), "2048/275/1102": (2048, 275, 1102)}
NORM = dict(signal_norm=True, symmetric_norm=True, max_norm=4.0, clip_norm=True, min_level_db=-100, ref_level_db=20,
            spec_gain=20, log_func="np.log10", power=1.5, preemphasis=0.0)


def signal(seconds, seed):
    """Harmonic-plus-noise: a gliding 6-partial tone under a syllable-rate envelope, with a little noise."""
    g = np.random.default_rng(seed)
    t = np.arange(int(SR * seconds)) / SR
    f0 = 110 + 60 * g.random()
    y = sum(np.sin(2 * np.pi * f0 * (k + 1) * (1 + 0.2 * np.sin(2 * np.pi * 0.7 * t)) * t) / (k + 1) for k in range(6))
    y = y * (0.55 + 0.45 * np.sin(2 * np.pi * (2 + g.random()) * t)) + 0.01 * g.standard_normal(t.size)
    return 0.3 * y


def normalised(y, n_fft, hop, win, mel):
    """The reference's forward chain (stft -> |.| -> [mel] -> amp_to_db -> normalize), float32 like the reference."""
    S = np.abs(G.stft(y, n_fft, hop, win)).astype(np.float32)
    if mel:
        S = np.dot(mel_filterbank(SR, n_fft, 80), S)
    D = 20 * np.log10(np.maximum(1e-5, S)) - NORM["ref_level_db"]
    S = ((D - NORM["min_level_db"]) / -NORM["min_level_db"]) * 2 * NORM["max_norm"] - NORM["max_norm"]
    return np.clip(S, -NORM["max_norm"], NORM["max_norm"]).astype(np.float32)


def ap_for(geom, iters, mel=True, **over):
    n_fft, hop, win = GEOM[geom]
    kw = dict(NORM, sample_rate=SR, num_mels=80, fft_size=n_fft, hop_length=hop, win_length=win, griffin_lim_iters=iters)
    kw.update(over)
    return kw


def oracle_dict(kw):
    d = dict(kw)
    d["base"] = np.e if d["log_func"] == "np.log" else 10
    return d


def run_gpu(kw, S, mel, u):
    ap = AudioProcessor(verbose=False, **kw)
    x = torch.from_numpy(S).to(DEV)
    uu = torch.from_numpy(u.astype(np.float32)).to(DEV)
    f = ap.inv_melspectrogram if mel else ap.inv_spectrogram
    return f(x, angles=uu).double().cpu().numpy()


def run_oracle(kw, S, mel, u, dtype=np.float64):
    basis = mel_filterbank(SR, kw["fft_size"], kw["num_mels"]) if mel else None
    return G.inv_spectrogram(S, oracle_dict(kw), u.astype(np.float32).astype(np.float64), basis, dtype)


@pytest.mark.parametrize("iters", [0, 1, 3])
@pytest.mark.parametrize("mel", [True, False], ids=["mel", "linear"])
@pytest.mark.parametrize("geom", sorted(GEOM))
def test_first_iterations_against_float64(geom, mel, iters):
    kw = ap_for(geom, iters)
    S = normalised(signal(2.0, 1), *GEOM[geom], mel)
    u = np.random.default_rng(2).random((GEOM[geom][0] // 2 + 1, S.shape[1]))
    got, want = run_gpu(kw, S, mel, u), run_oracle(kw, S, mel, u)
    assert got.shape == want.shape == (kw["hop_length"] * (S.shape[1] - 1),)
    assert G.rel_rms(got, want) <= 1e-5


@pytest.mark.parametrize("mel", [True, False], ids=["mel", "linear"])
@pytest.mark.parametrize("geom", sorted(GEOM))
def test_sixty_iterations_against_float32_and_float64(geom, mel):
    n_fft, hop, win = GEOM[geom]
    kw = ap_for(geom, 60)
    S = normalised(signal(2.5, 3), n_fft, hop, win, mel)
    u = np.random.default_rng(4).random((n_fft // 2 + 1, S.shape[1]))
    got = run_gpu(kw, S, mel, u)
    want = run_oracle(kw, S, mel, u)
    want32 = run_oracle(kw, S, mel, u, np.float32)
    err, err32 = G.rel_rms(got, want), G.rel_rms(want32, want)
    assert err <= 4 * err32 + 1e-6 and err <= 1e-4, (err, err32)
    basis = mel_filterbank(SR, n_fft, 80) if mel else None
    target = G.magnitudes(S, oracle_dict(kw), basis).astype(np.float64)
    sc_got = G.spectral_convergence(got, target, n_fft, hop, win)
    sc_want = G.spectral_convergence(want, target, n_fft, hop, win)
    assert abs(sc_got - sc_want) <= 1e-4 * sc_want, (sc_got, sc_want)


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("mel", [True, False], ids=["mel", "linear"])
def test_cpu_suite_cases(case, mel, tmp_path):
    kw = dict(CASES[case])
    stats = kw.pop("stats", False)
    ap_kw = {k: v for k, v in BASE_AP.items()}
    ap_kw.update(kw)
    C = ap_kw["num_mels"] if mel else ap_kw["fft_size"] // 2 + 1
    S = inputs(CASES[case], C, 40, seed=8)
    u = np.random.default_rng(9).random((ap_kw["fft_size"] // 2 + 1, 40))
    od = oracle_ap(CASES[case])
    if stats:
        st, ap_kw["stats_path"] = stats_for(ap_kw, tmp_path)
        od["stats"] = {"mel": (st["mel_mean"], st["mel_std"]), "linear": (st["linear_mean"], st["linear_std"])}
    ap = AudioProcessor(verbose=False, **ap_kw)
    f = ap.inv_melspectrogram if mel else ap.inv_spectrogram
    x, uu = torch.from_numpy(S).to(DEV), torch.from_numpy(u.astype(np.float32)).to(DEV)
    basis = mel_filterbank(ap_kw["sample_rate"], ap_kw["fft_size"], ap_kw["num_mels"]) if mel else None
    if stats and not mel:
        with pytest.raises(RuntimeError, match="Mean-Var"):
            f(x, angles=uu)
        return
    got = f(x, angles=uu).double().cpu().numpy()
    want = G.inv_spectrogram(S, od, u.astype(np.float32).astype(np.float64), basis)
    assert got.shape == want.shape
    assert G.rel_rms(got, want) <= 1e-5


def test_deemphasis_against_lfilter():
    # 400 frames x hop 256 = 102 144 samples through the chunked scan
    kw = ap_for("1024/256/1024", 0, preemphasis=0.97)
    S = normalised(signal(4.7, 5), 1024, 256, 1024, True)[:, :400]
    u = np.random.default_rng(6).random((513, 400))
    plain = run_gpu(dict(kw, preemphasis=0.0), S, True, u)
    got = run_gpu(kw, S, True, u)
    assert got.shape[0] >= 100000
    want = scipy.signal.lfilter([1], [1, -0.97], plain)
    assert G.rel_rms(got, want) <= 1e-5


def ragged(B=33, seed=10):
    g = np.random.default_rng(seed)
    lens = np.concatenate([[2, 800], g.integers(2, 801, B - 2)])
    T = int(lens.max())
    S = normalised(signal(T * 256 / SR + 0.05, 11), 1024, 256, 1024, True)[:, :T]
    x = np.stack([np.roll(S, 37 * b, axis=1) for b in range(B)])          # [B, 80, T]
    u = g.random((B, 513, T)).astype(np.float32)
    return x, lens, u


def test_ragged_batch_equals_single_rows_and_apply_griffin_lim():
    ap = AudioProcessor(verbose=False, **ap_for("1024/256/1024", 4))
    x, lens, u = ragged()
    X, U = torch.from_numpy(x).to(DEV), torch.from_numpy(u).to(DEV)
    wav, wl = ap.inv_melspectrogram(X, lengths=torch.from_numpy(lens), angles=U)
    assert wl.tolist() == [256 * (int(n) - 1) for n in lens]
    for b, n in enumerate(lens):
        one = ap.inv_melspectrogram(X[b, :, :n], angles=U[b, :, :n])
        assert torch.equal(wav[b, : 256 * (n - 1)], one), b
        assert float(wav[b, 256 * (n - 1):].abs().sum()) == 0.0
    # [B, T, C] input (time_last=False) gives the same result
    wav_t, _ = ap.inv_melspectrogram(X.transpose(1, 2), lengths=torch.from_numpy(lens), angles=U, time_last=False)
    assert torch.equal(wav_t, wav)

    # apply_griffin_lim: every row on its full padded spectrogram, then trimmed
    class Cfg:
        model = "glow_tts"

    full, _ = ap.inv_melspectrogram(X[:5], angles=U[:5])
    wavs = apply_griffin_lim(X[:5].transpose(1, 2), torch.from_numpy(lens[:5]), Cfg, ap, angles=U[:5])
    for b in range(5):
        assert torch.equal(wavs[b], full[b, : int(lens[b]) * 256 - 256])


def test_default_draws_follow_numpy_seed():
    kw = ap_for("1024/256/1024", 3)
    ap = AudioProcessor(verbose=False, **kw)
    S = normalised(signal(1.0, 12), 1024, 256, 1024, True)
    np.random.seed(21)
    got = ap.inv_melspectrogram(torch.from_numpy(S).to(DEV)).double().cpu().numpy()
    np.random.seed(21)
    u = np.random.rand(513, S.shape[1])
    want = G.inv_spectrogram(S, oracle_dict(kw), u, mel_filterbank(SR, 1024, 80))
    assert G.rel_rms(got, want) <= 1e-5


def test_non_finite_row_gives_one_zero_sample():
    ap = AudioProcessor(verbose=False, **ap_for("1024/256/1024", 3, signal_norm=False))
    x, lens, u = ragged(B=3, seed=13)
    x = np.clip(x, -4, 4) * 5 - 40          # dB, without normalisation
    X, U = torch.from_numpy(x).to(DEV), torch.from_numpy(u).to(DEV)
    good, gl = ap.inv_melspectrogram(X, lengths=torch.from_numpy(lens), angles=U)
    X[1, 3, 5] = float("inf")
    wav, wl = ap.inv_melspectrogram(X, lengths=torch.from_numpy(lens), angles=U)
    assert wl.tolist() == [gl[0].item(), 1, gl[2].item()]
    assert float(wav[1].abs().sum()) == 0.0
    assert torch.equal(wav[0], good[0]) and torch.equal(wav[2], good[2])
    one = ap.inv_melspectrogram(X[1, :, : lens[1]], angles=U[1, :, : lens[1]])
    assert one.shape == (1,) and float(one[0]) == 0.0


@pytest.mark.parametrize("mel", [True, False], ids=["mel", "linear"])
def test_repeatable_over_poisoned_workspace_and_dispatch(mel):
    ap = AudioProcessor(verbose=False, **ap_for("1024/256/1024", 5, preemphasis=0.97))
    x, lens, u = ragged(B=4, seed=14)
    if not mel:
        x = np.repeat(x[:, :1], 513, axis=1) - np.linspace(0, 2, 513, dtype=np.float32)[None, :, None]
    X, U, Lt = torch.from_numpy(x).to(DEV), torch.from_numpy(u).to(DEV), torch.from_numpy(lens)
    f = ap.inv_melspectrogram if mel else ap.inv_spectrogram
    first, _ = f(X, lengths=Lt, angles=U)
    _lib.workspace(DEV, 1, "griffin_lim").fill_(255)    # NaN bit patterns everywhere
    with _lib.dispatch_log() as log:
        again, _ = f(X, lengths=Lt, angles=U)
    assert torch.equal(first, again)
    prep = ["gl_prepare", "fma", "gl_prepare"] if mel else ["gl_prepare"]
    assert log.names == prep + ["gl_iter"] * 6 + ["gl_deemphasis"], log.names


@pytest.mark.parametrize("time_last", [True, False], ids=["BCT", "BTC"])
@pytest.mark.parametrize("mel", [True, False], ids=["mel", "linear"])
def test_layout_is_explicit_when_frames_equal_channels(mel, time_last):
    # T == C: the shape alone cannot tell [B, C, T] from [B, T, C]; the result must follow time_last, and equal the
    # oracle on the row read the stated way
    kw = ap_for("1024/256/1024", 2)
    C = 80 if mel else 513
    g = np.random.default_rng(15)
    x = g.uniform(-4, 4, (2, C, C)).astype(np.float32)         # rows as [C, T]
    u = g.random((2, 513, C)).astype(np.float32)
    lens = np.array([C, 41])
    ap = AudioProcessor(verbose=False, **kw)
    f = ap.inv_melspectrogram if mel else ap.inv_spectrogram
    X = torch.from_numpy(x if time_last else np.ascontiguousarray(x.transpose(0, 2, 1))).to(DEV)
    wav, wl = f(X, lengths=torch.from_numpy(lens), angles=torch.from_numpy(u).to(DEV), time_last=time_last)
    basis = mel_filterbank(SR, 1024, 80) if mel else None
    for b in range(2):
        n = int(lens[b])
        want = G.inv_spectrogram(x[b, :, :n], oracle_dict(kw), u[b, :, :n].astype(np.float64), basis)
        assert int(wl[b]) == want.shape[0]
        assert G.rel_rms(wav[b, :n * 256 - 256].double().cpu().numpy(), want) <= 1e-5
    # the channel axis is checked against the stated layout
    with pytest.raises(ValueError, match="channel axis"):
        f(X[:, :, :40] if time_last else X[:, :40, :], time_last=not time_last)


def test_tacotron_linear_chain():
    from test_tacotron_gpu import make, tokens

    cfg, model, _ = make(max_decoder_steps=30, out_channels=513)
    text, lens = tokens([9, 5])
    out = model.inference(text.to(DEV), {"x_lengths": lens.to(DEV)})
    y, ylen = out["model_outputs"], out["model_outputs_len"]       # [B, T, 513] on the device
    kw = ap_for("1024/256/1024", 3)
    ap = AudioProcessor(verbose=False, **kw)
    u = torch.rand(2, 513, y.shape[1], generator=torch.Generator().manual_seed(3)).to(DEV)
    wav, wl = ap.inv_spectrogram(y, lengths=ylen, angles=u, time_last=False)
    for b in range(2):
        n = int(ylen[b])
        want = G.inv_spectrogram(y[b, :n].T.contiguous().cpu().numpy(), oracle_dict(kw), u[b, :, :n].cpu().double().numpy())
        assert int(wl[b]) == want.shape[0]
        assert G.rel_rms(wav[b, : want.shape[0]].cpu().numpy(), want) <= 1e-5


def test_glow_tts_mel_chain():
    # GlowTTS.inference's model_outputs: a transposed [B, T, C] view with int64 y_lengths, straight into Griffin-Lim
    from test_glow_oracle_cpu import run_case
    from tts_b200.glow_tts import GlowTTS

    cfg, sd, x, lens, _, _ = run_case("default")
    m = GlowTTS(cfg).eval()
    m.load_state_dict(sd)
    out = m.to(DEV).inference(x.to(DEV), {"x_lengths": lens.to(DEV)})
    mel, ylen = out["model_outputs"], out["y_lengths"]
    assert not mel.is_contiguous()
    C = mel.shape[2]
    kw = dict(ap_for("1024/256/1024", 3), num_mels=C, signal_norm=False)   # Glow-TTS mels are log amplitudes
    kw.update(log_func="np.log", spec_gain=1)
    ap = AudioProcessor(verbose=False, **kw)
    u = torch.rand(mel.shape[0], 513, mel.shape[1], generator=torch.Generator().manual_seed(4)).to(DEV)
    wav, wl = ap.inv_melspectrogram(mel, lengths=ylen, angles=u, time_last=False)
    for b in range(mel.shape[0]):
        n = int(ylen[b])
        S = mel[b, :n].T.contiguous().cpu().numpy()
        want = G.inv_spectrogram(S, oracle_dict(kw), u[b, :, :n].cpu().double().numpy(), mel_filterbank(SR, 1024, C))
        assert int(wl[b]) == want.shape[0] == 256 * (n - 1)
        assert G.rel_rms(wav[b, : want.shape[0]].cpu().numpy(), want) <= 1e-5


def test_rejections():
    x = torch.zeros(80, 10, device=DEV)
    with pytest.raises(NotImplementedError):
        AudioProcessor(verbose=False, **ap_for("1024/256/1024", 1, fft_size=1000, win_length=1000)).inv_melspectrogram(x)
    with pytest.raises(NotImplementedError):
        AudioProcessor(verbose=False, **ap_for("1024/256/1024", 1, stft_pad_mode="constant")).inv_melspectrogram(x)
    ap = AudioProcessor(verbose=False, **ap_for("1024/256/1024", 1))
    with pytest.raises(ValueError):
        ap.inv_melspectrogram(x[:, :1])
    with pytest.raises(ValueError):
        ap.inv_melspectrogram(x.expand(2, 80, 10), lengths=torch.tensor([10, 1]))
    with pytest.raises(RuntimeError, match="no CPU path"):
        ap.inv_melspectrogram(x.cpu())
    with pytest.raises(RuntimeError, match="no CPU path"):
        griffin_lim(spec=torch.ones(513, 4), num_iter=1, hop_length=256, win_length=1024, fft_size=1024)
