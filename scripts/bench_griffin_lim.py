"""Griffin-Lim benchmark: ``AudioProcessor.inv_melspectrogram`` on a ragged batch (32 rows of 400-860 frames, 80 mels ->
513 bins, n_fft 1024 / hop 256 / win 1024, 60 iterations), against torch-eager batched Griffin-Lim (torch.stft / istft,
float32) on the same GPU, per call and per frame (eager runs the padded batch), and the reference's float64 per-row
loop (the oracle) on the host for the first rows.
Prints one JSON line: ms per call (CUDA events), the iteration kernel's time (torch.profiler, a run of its own), its
FLOP/s and bytes/s from counts computed here, the speed-up over eager, the GPU output's relative RMS against eager, and
the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tts_b200.audio import AudioProcessor, mel_filterbank  # noqa: E402

N_FFT, HOP, WIN, MELS, ITERS, SR = 1024, 256, 1024, 80, 60, 22050


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:   # noqa: BLE001 -- the name still comes from torch
        return torch.cuda.get_device_name(0), "unknown"


def workload(B, seed=0):
    g = np.random.default_rng(seed)
    lens = g.integers(400, 861, B)
    T = int(lens.max())
    x = g.uniform(-4, 4, (B, MELS, T)).astype(np.float32)
    t = np.arange(T)[None, None, :]
    x = np.clip(x * 0.3 + np.sin(t / 7.0 + np.arange(MELS)[None, :, None] / 5.0) * 2 - 1, -4, 4).astype(np.float32)
    u = g.random((B, N_FFT // 2 + 1, T)).astype(np.float32)
    return x, lens, u


def counts(lens):
    """FLOPs and HBM bytes of the iteration kernels, from shapes: per frame-iteration two real n_fft-point FFTs
    (5 n log2 n / 2 each, as half a complex FFT), the projection (~20 flops per bin), the window and overlap-add;
    bytes: one |S| row read plus the waveform span read and written."""
    F = N_FFT // 2 + 1
    frames = int(np.sum(lens))
    fft = 2 * (5 * N_FFT * np.log2(N_FFT) / 2)
    flop_per = fft + 20 * F + 4 * N_FFT
    bytes_per = 4 * F + 2 * 4 * HOP
    return frames * ITERS * flop_per, frames * ITERS * bytes_per


def eager(mag, lens_t, u, iters):
    """Batched float32 Griffin-Lim with torch.stft / istft on the padded batch (the rows' tails are zero magnitudes)."""
    w = torch.hann_window(WIN, device=mag.device)
    S = mag.to(torch.complex64)
    y = torch.istft(S * torch.exp(2j * np.pi * u.to(torch.float32)), N_FFT, HOP, WIN, window=w, center=True)
    for _ in range(iters):
        X = torch.stft(y, N_FFT, HOP, WIN, window=w, center=True, pad_mode="reflect", return_complex=True)
        y = torch.istft(S * torch.exp(1j * torch.angle(X)), N_FFT, HOP, WIN, window=w, center=True)
    return y


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--rows", type=int, default=32)
    ap_.add_argument("--reps", type=int, default=10)
    ap_.add_argument("--oracle-rows", type=int, default=2)
    ap_.add_argument("--profile", action="store_true", help="time the iteration kernel with torch.profiler only")
    args = ap_.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_griffin_lim: needs a CUDA device")
    dev = torch.device("cuda:0")
    ap = AudioProcessor(verbose=False, sample_rate=SR, num_mels=MELS, fft_size=N_FFT, hop_length=HOP, win_length=WIN,
                        griffin_lim_iters=ITERS, power=1.5, signal_norm=True, symmetric_norm=True, max_norm=4.0,
                        clip_norm=True, min_level_db=-100, ref_level_db=20)
    x, lens, u = workload(args.rows)
    X, U, Lt = torch.from_numpy(x).to(dev), torch.from_numpy(u).to(dev), torch.from_numpy(lens)
    call = lambda: ap.inv_melspectrogram(X, lengths=Lt, angles=U)   # noqa: E731
    for _ in range(2):
        wav, wl = call()
    torch.cuda.synchronize()

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        iter_us = [e.device_time for e in prof.events() if "gl_iter_kernel" in e.name]
        other = {e.name.split("(")[0][-40:]: e.device_time for e in prof.events() if "gl_" in e.name and
                 "gl_iter_kernel" not in e.name}
        flop, byts = counts(lens)
        mean_us = float(np.mean(iter_us[1:]))
        print(json.dumps({"metric": "griffin_lim_iter_kernel", "iter_kernels": len(iter_us),
                          "iter_kernel_us_mean": round(mean_us, 2), "first_istft_us": round(iter_us[0], 2),
                          "other_kernels_us": {k: round(v, 2) for k, v in other.items()},
                          "iter_tflops": round(flop / ITERS / (mean_us * 1e-6) / 1e12, 2),
                          "iter_hbm_gbs": round(byts / ITERS / (mean_us * 1e-6) / 1e9, 1),
                          "gpu": card()[0], "power_limit": card()[1]}))
        return

    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.reps):
        call()
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / args.reps

    # torch eager on the same magnitudes (the fused path's own prepare output, recomputed here in torch)
    basis = torch.from_numpy(np.linalg.pinv(mel_filterbank(SR, N_FFT, MELS))).to(dev)
    D = ((X.clamp(-4, 4) + 4) * 100 / 8 - 100) + 20
    mag = torch.clamp(basis @ torch.pow(10.0, D / 20), min=1e-10) ** 1.5
    mag = mag * (torch.arange(mag.shape[-1], device=dev)[None, None, :] < Lt.to(dev)[:, None, None])
    eager(mag, Lt, U, 2)
    torch.cuda.synchronize()
    start.record()
    reps_e = max(1, args.reps // 2)
    for _ in range(reps_e):
        ye = eager(mag, Lt, U, ITERS)
    end.record()
    torch.cuda.synchronize()
    ms_eager = start.elapsed_time(end) / reps_e
    # the eager batch shares the padded length, so only rows of full length are comparable sample for sample
    b = int(np.argmax(lens))
    n = int(wl[b])
    d = (wav[b, :n].double() - ye[b, :n].double())
    rel_eager = float(d.pow(2).mean().sqrt() / ye[b, :n].double().pow(2).mean().sqrt())

    # the reference's way: one row at a time in float64 on the host
    import griffin_lim_oracle as G

    kw = dict(signal_norm=True, symmetric_norm=True, max_norm=4.0, clip_norm=True, min_level_db=-100, ref_level_db=20,
              spec_gain=20.0, base=10, power=1.5, griffin_lim_iters=ITERS, hop_length=HOP, win_length=WIN,
              preemphasis=0.0)
    fb = mel_filterbank(SR, N_FFT, MELS)
    t0 = time.perf_counter()
    rel_oracle = []
    for r in range(args.oracle_rows):
        n_r = int(lens[r])
        want = G.inv_spectrogram(x[r, :, :n_r], kw, u[r, :, :n_r].astype(np.float64), fb)
        rel_oracle.append(G.rel_rms(wav[r, : want.shape[0]].cpu().numpy(), want))
    host_s_per_row = (time.perf_counter() - t0) / max(1, args.oracle_rows)

    flop, byts = counts(lens)
    name, limit = card()
    # eager transforms the padded batch (rows x T_max frames), the fused chain only each row's own frames: compare
    # per frame as well as per call
    eager_frames = args.rows * int(lens.max())
    print(json.dumps({
        "metric": "griffin_lim_inv_melspectrogram", "rows": args.rows, "frames": int(lens.sum()), "iters": ITERS,
        "ms_per_call": round(ms, 3), "torch_eager_ms_per_call": round(ms_eager, 3),
        "speedup_vs_eager": round(ms_eager / ms, 2), "eager_frames": eager_frames,
        "us_per_frame": round(1e3 * ms / int(lens.sum()), 4),
        "torch_eager_us_per_frame": round(1e3 * ms_eager / eager_frames, 4),
        "speedup_vs_eager_per_frame": round((ms_eager / eager_frames) / (ms / int(lens.sum())), 2),
        "call_tflops": round(flop / (ms * 1e-3) / 1e12, 2), "call_hbm_gbs": round(byts / (ms * 1e-3) / 1e9, 1),
        "rel_rms_vs_eager_longest_row": rel_eager,
        "host_float64_s_per_row": round(host_s_per_row, 3), "rel_rms_vs_float64_oracle": rel_oracle,
        "gpu": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
