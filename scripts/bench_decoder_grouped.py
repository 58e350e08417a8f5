#!/usr/bin/env python
"""The decoder's 32- and 64-channel ResBlock convs (the `tc3_grouped` dispatch, split fp16) at bench.py's length, layer by
layer.  Prints one JSON line.

  python scripts/bench_decoder_grouped.py [--batch 32] [--frames 192] [--steps 20]

For every distinct conv shape of the last two decoder stages of bench.py's model (dense, `batch` rows of `frames`
decoder frames, so the stages run at 64 x and 128 x `frames` columns), the three forms a ResBlock runs are timed:
c1 (leaky ReLU in, no residual), c2 + residual, and the last c2 + residual + accumulate into the MRF sum + final divide.
Each timed launch follows a 256 MiB L2-evicting write outside the CUDA events, and the forms alternate round by round;
the median ms per launch is reported.  Beside it: the algorithmic FLOPs and HBM bytes from the shape, the MMA floor
(3 fp16 MMAs per multiply-add at the data sheet's dense 989 TFLOP/s), the HBM floor (bytes at 3.35 TB/s) and the larger
of the two over the measured time.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402  (the headline workload's model)
from bench_stream import card  # noqa: E402

MMA_PEAK = 989e12          # H100 SXM data sheet, dense FP16
HBM_PEAK = 3.35e12         # H100 SXM data sheet, HBM3
SLOPE = 0.1                # the ResBlocks' leaky ReLU
FORMS = ("c1", "c2_res", "c2_res_acc")


def grouped_shapes(cfg):
    """(stage, channels, k, dil, frame_rate) of the ResBlock convs of the stages with 32 / 64 channels."""
    out, ch, rate = [], cfg["upsample_initial_channel"], 1
    for s, u in enumerate(cfg["upsample_factors"]):
        ch, rate = ch // 2, rate * u
        if ch not in (32, 64):
            continue
        shapes = {(rk, dd) for rk, dils in zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])
                  for d in dils for dd in (d, 1)}              # ResBlock1: convs1 at dilation d, convs2 at 1
        out += [(s, ch, rk, dd, rate) for rk, dd in sorted(shapes)]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=192)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_decoder_grouped.py needs a CUDA device: there is no CPU fallback"
    from tts_b200 import _lib
    from tts_b200.conv import FusedConv1d
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = bench.build_model().waveform_decoder._cfg
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    gen = torch.Generator().manual_seed(0)
    line = {"metric": "decoder_grouped_convs", "card": card(0), "batch": args.batch, "frames": args.frames,
            "steps": args.steps, "layers": []}
    for s, ch, k, dil, rate in grouped_shapes(cfg):
        t = args.frames * rate
        w = torch.randn(ch, ch, k, generator=gen, dtype=torch.float64) / (ch * k) ** 0.5
        conv = FusedConv1d(w, torch.zeros(ch, dtype=torch.float64), dilation=dil, padding=dil * (k - 1) // 2,
                           precision="f16x3")
        x, r, acc = (torch.randn(args.batch, ch, t, device=dev) for _ in range(3))
        calls = {"c1": lambda: conv(x, in_slope=SLOPE),
                 "c2_res": lambda: conv(x, in_slope=SLOPE, residual=r),
                 "c2_res_acc": lambda: conv(x, in_slope=SLOPE, residual=r, accumulate_into=acc, post_div=3.0)}
        with _lib.dispatch_log() as log:
            for f in FORMS:
                calls[f]()
        torch.cuda.synchronize()
        times = {f: [] for f in FORMS}
        for _ in range(args.steps):
            for f in FORMS:
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                calls[f]()
                e1.record()
                e1.synchronize()
                times[f].append(e0.elapsed_time(e1))
        assert _lib.lib().b200tts_debug_tc_error() == 0
        tensor = args.batch * ch * t * 4
        flop = 2.0 * args.batch * t * ch * ch * k
        for f in FORMS:
            nbytes = tensor * {"c1": 2, "c2_res": 3, "c2_res_acc": 4}[f]
            ms = statistics.median(times[f])
            mma_ms, hbm_ms = 3 * flop / MMA_PEAK * 1e3, nbytes / HBM_PEAK * 1e3
            line["layers"].append({"stage": s, "channels": ch, "k": k, "dil": dil, "T": t, "form": f,
                                   "dispatch": log.names[FORMS.index(f)], "ms": round(ms, 4),
                                   "ms_min": round(min(times[f]), 4), "ms_max": round(max(times[f]), 4),
                                   "gflop": round(flop / 1e9, 2), "mbytes": round(nbytes / 1e6, 1),
                                   "mma_floor_ms": round(mma_ms, 4), "hbm_floor_ms": round(hbm_ms, 4),
                                   "floor_share": round(max(mma_ms, hbm_ms) / ms, 3)})
    # what one decoder step runs per stage: ResBlock (kernel rk, dilations dils) = c1 at every d, c2 + residual after all
    # but the last, and the last c2 writes (first ResBlock) or accumulates into (the others) the MRF sum
    ms = {(d["stage"], d["k"], d["dil"], d["form"]): d["ms"] for d in line["layers"]}
    stages = {}
    for s in sorted({d["stage"] for d in line["layers"]}):
        tot = 0.0
        for i, (rk, dils) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            tot += sum(ms[(s, rk, d, "c1")] for d in dils) + (len(dils) - 1) * ms[(s, rk, 1, "c2_res")]
            tot += ms[(s, rk, 1, "c2_res" if i == 0 else "c2_res_acc")]
        stages[f"stage{s}"] = round(tot, 3)
    line["dense_stage_ms"] = stages
    print(json.dumps(line))


if __name__ == "__main__":
    main()
