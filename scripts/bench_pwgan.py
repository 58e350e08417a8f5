"""Parallel WaveGAN generator throughput on the MelGAN bench batch (32 utterances of 384 frames, 12 288 frames), inference
with supplied noise: 32 x 388 x 256 = 3 178 496 output samples per call.

Reports the CUDA-event time per call and audio samples/s; from torch.profiler in a run of its own, the kernel time of the
whole call and of the residual stack alone (the 30 pwgan_layer_kernel launches), the stack's share of it and its
achieved TFLOP/s and GB/s against the work counted from shapes; the oracle (tests/pwgan_oracle.py, the reference's layer
sequence) in torch eager on the same GPU with TF32 off and on the host CPU (4 of the 32 utterances, with the thread count); parity against the eager GPU run; the card's name and
power limit, read in the same run.  Writes nothing; prints one JSON line.

    python scripts/bench_pwgan.py [--iters N]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

B, FRAMES, PAD, HOP, LAYERS = 32, 384, 2, 256, 30
MMA_FLOP_PER_SAMPLE_LAYER = 2 * 128 * 64 * 3 + 2 * 128 * 64     # gate conv + out|skip 1x1: 65 536
HBM_BYTES_PER_SAMPLE_LAYER = 64 * 4 * (1 + 1 + 2)               # x read, x_new write, skip read-modify-write: 1 024


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def event_time(fn, iters):
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pwgan: needs a CUDA device")
    import pwgan_oracle as PO
    from ref_golden import layout, seeded_state_dict
    from tts_b200.pwgan import ParallelWaveganGenerator

    dev = torch.device("cuda:0")
    name, limit = card()
    model = ParallelWaveganGenerator().eval()
    sd = seeded_state_dict(layout(model.state_dict()), 0)
    model.load_state_dict(sd)
    model.to(dev)
    g = torch.Generator().manual_seed(0)
    c = torch.randn(B, 80, FRAMES, generator=g)
    tf = FRAMES + 2 * PAD
    samples = B * tf * HOP
    noise = torch.randn(B, 1, tf * HOP, generator=g)
    c_dev, noise_dev = c.to(dev), noise.to(dev)

    call_ms = event_time(lambda: model.inference(c_dev, noise=noise_dev), args.iters)
    got = model.inference(c_dev, noise=noise_dev)

    # the residual stack alone: kernel time of the fused layer launches, in a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.inference(c_dev, noise=noise_dev)
        torch.cuda.synchronize()
    events = prof.key_averages()
    stack_us = sum(e.self_device_time_total for e in events if "pwgan_layer_kernel" in e.key)
    kernels_us = sum(e.self_device_time_total for e in events)   # every kernel of the profiled call
    stack_s = stack_us * 1e-6
    flop = samples * LAYERS * MMA_FLOP_PER_SAMPLE_LAYER
    nbytes = samples * LAYERS * HBM_BYTES_PER_SAMPLE_LAYER

    # the oracle in torch eager on the same GPU, fp32 without TF32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    with torch.no_grad():
        eager = lambda: PO.inference(sd_dev, c_dev, noise_dev)   # noqa: E731
        eager_ms = event_time(eager, max(1, args.iters // 2))
        want = eager()
    rel = float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())

    # host CPU, 4 utterances
    nb = 4
    with torch.no_grad():
        t0 = time.perf_counter()
        PO.inference(sd, c[:nb], noise[:nb])
        cpu_s = time.perf_counter() - t0

    print(json.dumps({
        "workload": f"PWGAN inference, {B} x {FRAMES} frames (+{PAD} replicate pad each side), supplied noise",
        "card": name, "power_limit": limit,
        "call_ms": round(call_ms, 3), "samples_per_s": round(samples / (call_ms * 1e-3)),
        "profiled_call_kernel_ms": round(kernels_us * 1e-3, 3),
        "residual_stack_ms": round(stack_s * 1e3, 3),
        "residual_stack_share_of_profiled_kernels": round(stack_us / kernels_us, 3),
        "residual_stack_tflops": round(flop / stack_s / 1e12, 1),
        "residual_stack_gbps": round(nbytes / stack_s / 1e9, 1),
        "counted_stack_tflop": round(flop / 1e12, 2), "counted_stack_gb": round(nbytes / 1e9, 1),
        "bound_mma_ms_at_989_over_3_tflops": round(flop / (989e12 / 3) * 1e3, 1),
        "bound_hbm_ms_at_3350_gbps": round(nbytes / 3.35e12 * 1e3, 1),
        "eager_gpu_fp32_ms": round(eager_ms, 3), "speedup_vs_eager_gpu": round(eager_ms / call_ms, 2),
        "cpu_4_utterances_s": round(cpu_s, 3), "cpu_threads": torch.get_num_threads(),
        "rel_rms_vs_eager_gpu": rel,
    }))


if __name__ == "__main__":
    main()
