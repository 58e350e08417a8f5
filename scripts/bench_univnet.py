"""UnivNet generator throughput on the MelGAN bench batch (32 utterances of 384 frames, 12 288 frames), inference with
supplied noise: 32 x 384 x 256 = 3 145 728 output samples per call, with the zoo model's shape (hidden 32, factors
[8, 8, 4], 4 LVC layers per block, KPnet hidden 64, kernel 3).

Reports the CUDA-event time per call and audio samples/s; from torch.profiler in a run of its own, the kernel time of the
prediction GEMMs (univnet_predict_kernel), of the LVC layers (univnet_lvc_kernel) and of the rest, the first two with
achieved TFLOP/s and GB/s against the work counted from shapes below; the oracle (tests/univnet_oracle.py) in torch eager
on the same GPU with TF32 off, and parity against it; the card's name and power limit, read in the same run.  Writes
nothing; prints one JSON line.

    python scripts/bench_univnet.py [--iters N]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

B, FRAMES, FACTORS, LAYERS, KP_H, KP_K, MELS, C = 32, 384, (8, 8, 4), 4, 64, 3, 80, 32
HOPS = (8, 64, 256)
SAMPLES_ALL_BLOCKS = B * FRAMES * sum(HOPS)                     # samples the LVC layers run on: 4 030 464
LVC_FLOP_PER_SAMPLE_LAYER = 2 * C * 3 * C + 2 * 2 * C * 3 * C   # conv_i 6 144 + LVC 12 288
LVC_X_BYTES_PER_SAMPLE_LAYER = 2 * C * 4                        # x read + x written: 256
MP = LAYERS * (2 * C * 3 * C + 2 * C)                           # predicted floats per frame and block: 24 832
PRED_GEMM_FLOP_PER_FRAME = 2 * MP * KP_H * KP_K                 # kernel_conv | bias_conv: 9.54 M
KPNET_FLOP_PER_FRAME = 2 * (MELS * KP_H * 5 + 6 * KP_H * KP_H * KP_K)


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
        raise SystemExit("bench_univnet: needs a CUDA device")
    import univnet_oracle as UO
    from ref_golden import layout, seeded_state_dict
    from tts_b200.univnet import UnivnetGenerator

    dev = torch.device("cuda:0")
    name, limit = card()
    model = UnivnetGenerator(in_channels=64, out_channels=1, hidden_channels=C, cond_channels=MELS,
                             upsample_factors=list(FACTORS), lvc_layers_each_block=LAYERS, lvc_kernel_size=3,
                             kpnet_hidden_channels=KP_H, kpnet_conv_size=KP_K, dropout=0.0).eval()
    sd = seeded_state_dict(layout(model.state_dict()), 0)
    model.load_state_dict(sd)
    model.to(dev)
    g = torch.Generator().manual_seed(0)
    c = torch.randn(B, MELS, FRAMES, generator=g)
    noise = torch.randn(B, 64, FRAMES, generator=g)
    c_dev, noise_dev = c.to(dev), noise.to(dev)
    samples = B * FRAMES * HOPS[-1]

    call_ms = event_time(lambda: model.inference(c_dev, noise=noise_dev), args.iters)
    got = model.inference(c_dev, noise=noise_dev)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.inference(c_dev, noise=noise_dev)
        torch.cuda.synchronize()
    events = prof.key_averages()
    pred_us = sum(e.self_device_time_total for e in events if "univnet_predict_kernel" in e.key)
    lvc_us = sum(e.self_device_time_total for e in events if "univnet_lvc_kernel" in e.key)
    kernels_us = sum(e.self_device_time_total for e in events)
    frames_blocks = B * FRAMES * len(FACTORS)
    pred_flop = frames_blocks * PRED_GEMM_FLOP_PER_FRAME
    pred_bytes = frames_blocks * MP * 4                                  # the predicted kernels written, fp32
    lvc_flop = SAMPLES_ALL_BLOCKS * LAYERS * LVC_FLOP_PER_SAMPLE_LAYER
    lvc_x_bytes = SAMPLES_ALL_BLOCKS * LAYERS * LVC_X_BYTES_PER_SAMPLE_LAYER
    lvc_bytes = lvc_x_bytes + pred_bytes                                 # + each layer reading its kernels once
    pred_s, lvc_s = pred_us * 1e-6, lvc_us * 1e-6

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    with torch.no_grad():
        eager = lambda: UO.generator(sd_dev, c_dev, noise_dev)   # noqa: E731
        eager_ms = event_time(eager, max(1, args.iters // 2))
        want = eager()
    rel = float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())

    print(json.dumps({
        "workload": f"UnivNet inference, {B} x {FRAMES} frames, supplied noise",
        "card": name, "power_limit": limit,
        "call_ms": round(call_ms, 3), "samples_per_s": round(samples / (call_ms * 1e-3)),
        "profiled_call_kernel_ms": round(kernels_us * 1e-3, 3),
        "predict_gemm_ms": round(pred_s * 1e3, 3), "predict_gemm_tflops": round(pred_flop / pred_s / 1e12, 1),
        "predict_gemm_gbps": round(pred_bytes / pred_s / 1e9, 1),
        "lvc_layers_ms": round(lvc_s * 1e3, 3), "lvc_layers_tflops": round(lvc_flop / lvc_s / 1e12, 1),
        "lvc_layers_gbps": round(lvc_bytes / lvc_s / 1e9, 1),
        "rest_ms": round((kernels_us - pred_us - lvc_us) * 1e-3, 3),
        "counted_predict_gemm_tflop": round(pred_flop / 1e12, 3), "counted_kpnet_convs_tflop": round(
            frames_blocks * KPNET_FLOP_PER_FRAME / 1e12, 3),
        "counted_predict_gb": round(pred_bytes / 1e9, 2),
        "counted_lvc_tflop": round(lvc_flop / 1e12, 3), "counted_lvc_gb": round(lvc_bytes / 1e9, 2),
        "bound_lvc_mma_ms_at_989_over_3_tflops": round(lvc_flop / (989e12 / 3) * 1e3, 2),
        "bound_lvc_hbm_ms_at_3350_gbps": round(lvc_bytes / 3.35e12 * 1e3, 2),
        "bound_predict_mma_ms_at_989_over_3_tflops": round(pred_flop / (989e12 / 3) * 1e3, 2),
        "bound_predict_hbm_ms_at_3350_gbps": round(pred_bytes / 3.35e12 * 1e3, 2),
        "eager_gpu_fp32_ms": round(eager_ms, 3), "speedup_vs_eager_gpu": round(eager_ms / call_ms, 2),
        "rel_rms_vs_eager_gpu": rel,
    }))


if __name__ == "__main__":
    main()
