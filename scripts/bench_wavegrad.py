#!/usr/bin/env python
"""WaveGrad refinement on the GPU: the default WavegradConfig (50-step test schedule, seeded weights) at two shapes,
8 utterances x 256 frames (524 288 samples per call) and 1 x 256 frames (the Synthesizer call shape).

Reports per shape: time per inference and per step (CUDA events around whole calls, after warm-up), audio samples/s,
the achieved TFLOP/s of the convs (FLOPs counted from the layer shapes below), launches per step, and the same inference
of the fp32 oracle (tests/wavegrad_oracle.py) in torch eager on the same GPU with TF32 off, on the same inputs, with the
relative RMS between the two.  One refinement step of the oracle on the host CPU (1 x 256 frames only: the 8-utterance
step takes minutes there) is reported as a per-step time, not extrapolated.  The card's name and power limit are read
in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import wavegrad_oracle as WO  # noqa: E402
from ref_golden import layout, seeded_state_dict  # noqa: E402
from tts_b200 import _lib  # noqa: E402
from tts_b200 import wavegrad as W  # noqa: E402


def flops_per_forward(args, B, T):
    """2 * Cout * Cin * K * Lout * B over every conv of Wavegrad.forward (x_conv included)."""
    f = args.upsample_factors
    n = len(f)
    L = [int(np.prod(f)) * T]
    for df in reversed(f[1:]):
        L.append(L[-1] // df)
    tot = 2 * args.y_conv_channels * 1 * 5 * L[0]
    ic = args.y_conv_channels
    for i in range(n):
        oc = args.ublock_out_channels[n - 1 - i]
        tot += 2 * ic * ic * 3 * L[i] + 2 * 2 * oc * ic * 3 * L[i]                       # FiLM i
        if i + 1 < n:
            d = args.dblock_out_channels[i]
            tot += 2 * d * ic * L[i + 1] + 2 * d * ic * 3 * L[i + 1] + 2 * 2 * d * d * 3 * L[i + 1]   # DBlock i
            ic = d
    xc = args.x_conv_channels
    tot += 2 * xc * args.in_channels * 3 * T
    for j in range(n):
        h, Lu = args.ublock_out_channels[j], L[n - 1 - j]
        tot += 2 * h * xc * Lu + 2 * h * xc * 3 * Lu + 3 * 2 * h * h * 3 * Lu           # UBlock j
        xc = h
    tot += 2 * 1 * xc * 3 * L[0]
    return tot * B, 2 * args.x_conv_channels * args.in_channels * 3 * T * B   # (forward, its x_conv share)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:  # pragma: no cover
        return f"unavailable ({e})"


def time_call(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--eager-reps", type=int, default=1)
    ap.add_argument("--no-cpu", action="store_true", help="skip the host-CPU oracle step")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wavegrad.py measures on a GPU"
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    cfg = W.WavegradConfig()
    model = W.Wavegrad(cfg).eval()
    sd = seeded_state_dict(layout(model.state_dict()), 5)
    model.load_state_dict(sd)
    s = cfg.test_noise_schedule
    beta = np.linspace(s["min_val"], s["max_val"], s["num_steps"])
    model.compute_noise_level(beta)
    model.to(dev)
    sched = WO.schedule(beta)
    sdd = {k: v.to(dev) for k, v in sd.items()}
    N = len(beta)
    res = {"card": card(), "config": "WavegradConfig() defaults, 50-step test schedule", "shapes": []}
    for B, T in ((8, 256), (1, 256)):
        g = torch.Generator().manual_seed(1)
        spec = torch.randn(B, 80, T, generator=g).to(dev)
        L = model.hop_len * T
        y0 = torch.randn(B, 1, L, generator=g).to(dev)
        zs = torch.randn(N - 1, B, 1, L, generator=g).to(dev)
        run = lambda: model.inference(spec, init_noise=y0, step_noise=zs)   # noqa: E731
        out = run()
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        run()
        torch.cuda.synchronize()
        launches = _lib.launch_count() - n0
        ts = time_call(run, a.reps, a.warmup)
        t = min(ts)
        fl_fwd, fl_x = flops_per_forward(cfg.model_params, B, T)
        fl_inf = N * (fl_fwd - fl_x) + fl_x                                    # x_conv once per inference
        eager = lambda: WO.inference(sdd, spec, sched, cfg.model_params, init_noise=y0, step_noise=zs)   # noqa: E731
        want = eager()
        te = min(time_call(eager, a.eager_reps, 1))
        rel = ((out - want).double().pow(2).mean().sqrt() / want.double().pow(2).mean().sqrt()).item()
        r = {"B": B, "T_frames": T, "samples": B * L, "steps": N, "inference_s": t, "inference_s_all": ts,
             "step_ms": t / N * 1e3, "samples_per_s": B * L / t, "tflop_per_call": fl_inf / 1e12,
             "achieved_tflops": fl_inf / t / 1e12, "launches_per_step": (launches - 1) / N,
             "eager_fp32_inference_s": te, "speedup_vs_eager": te / t, "rel_rms_vs_eager": rel,
             "inside_unit_interval": (out.abs() < 1).float().mean().item()}
        if B == 1 and not a.no_cpu:
            sdc = {k: v.cpu() for k, v in sd.items()}
            yc, xc = y0.cpu(), spec.cpu()
            lvl = sched["noise_level"][N - 1].repeat(B)
            t0 = time.perf_counter()
            with torch.no_grad():
                WO.forward(sdc, yc, xc, lvl, cfg.model_params)
            r["cpu_oracle_step_s"] = time.perf_counter() - t0
            r["cpu_threads"] = torch.get_num_threads()
        res["shapes"].append(r)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    with torch.no_grad():
        main()
