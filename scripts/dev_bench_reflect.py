"""Cost of reflection padding in the conv engine: each MelGAN reflect-padded layer shape timed as the reflect-padded launch
and as the same layer zero-padded, alternately, on the same weights and input (16-byte aligned rows, so both take the
same kernel family: the reflect variant of the tensor-core kernel against the zero-padding one).  Prints one line per
shape and one JSON line with the card's name.

    python scripts/dev_bench_reflect.py [--reps 5] [--iters 20] [--precision fp32|bf16|fp16]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tts_b200 import _lib  # noqa: E402
from tts_b200.conv import FusedConv1d  # noqa: E402

# multi-band MelGAN (MultibandMelganConfig) at the Glow-TTS bench batch's length: 32 x 384 frames -> stages x8, x4, x2
SHAPES = [("pre384_k7", 80, 384, 7, 1, 1.0, 384), ("res192_d1", 192, 192, 3, 1, 0.2, 3072),
          ("res192_d27", 192, 192, 3, 27, 0.2, 3072), ("res96_d9", 96, 96, 3, 9, 0.2, 12288),
          ("res48_d3", 48, 48, 3, 3, 0.2, 24576)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--precision", default="fp32", help="operand precision of the tensor-core kernels")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    dev = torch.device("cuda:0")
    rows = []
    for name, cin, cout, k, d, slope, t in SHAPES:
        g = torch.Generator().manual_seed(1)
        w = (torch.rand(cout, cin, k, generator=g) * 2 - 1) / (cin * k) ** 0.5
        b = torch.randn(cout, generator=g) * 0.05
        pad = (k - 1) // 2 * d
        convs = {m: FusedConv1d(w, b, dilation=d, padding=pad, padding_mode=m, precision=args.precision)
                 for m in ("reflect", "zeros")}
        x = torch.randn(32, cin, t, device=dev)
        names = {}
        for m, conv in convs.items():
            with _lib.dispatch_log() as log:
                conv(x, in_slope=slope)
            names[m] = log.names
        times = {m: [] for m in convs}
        for _ in range(args.reps):
            for m, conv in convs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    conv(x, in_slope=slope)
                e1.record()
                torch.cuda.synchronize()
                times[m].append(e0.elapsed_time(e1) / args.iters)
        med = {m: sorted(v)[len(v) // 2] for m, v in times.items()}
        # kernel time alone (torch.profiler, CUDA activity): excludes any host-side gap between the launches
        kern = {}
        for m, conv in convs.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    conv(x, in_slope=slope)
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "conv1d" in e.name]
            kern[m] = sum(e.device_time for e in ev) / max(1, len(ev)) / 1e3
        row = {"shape": name, "T": t, "B": 32, "reflect_ms": round(med["reflect"], 4), "zeros_ms": round(med["zeros"], 4),
               "ratio": round(med["reflect"] / med["zeros"], 4), "kernel_reflect_ms": round(kern["reflect"], 4),
               "kernel_zeros_ms": round(kern["zeros"], 4), "kernel_ratio": round(kern["reflect"] / kern["zeros"], 4),
               "dispatch": names}
        print(row)
        rows.append(row)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "precision": args.precision, "rows": rows}))


if __name__ == "__main__":
    main()
