"""Speaker-encoder throughput: a seeded, dataset-shaped set of 16 kHz clips (1.5-8 s, as compute_embeddings.py sees
them) through ``ResNetSpeakerEncoder.compute_embeddings`` at the reference's defaults (10 windows of 250 frames).

Reports clips/s and the achieved TFLOP/s from shape-derived FLOPs (convs and linears, counted below), next to two
bars on the same clips: torch eager on the GPU (cuDNN, TF32 off) and torch on the CPU with every host thread.  Prints
the parity of the kernels against the eager GPU run, the card name and its power limit, then one JSON line.

    python scripts/bench_speaker_encoder.py [--clips 64] [--steps 5] [--warmup 2] [--cpu-clips 4]
"""
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
import encoder_oracle as EO  # noqa: E402
from tts_b200.encoder import ResNetSpeakerEncoder  # noqa: E402

AUDIO = dict(fft_size=512, win_length=400, hop_length=160, sample_rate=16000, preemphasis=0.97, num_mels=64)
KW = dict(encoder_type="ASP", log_input=True, use_torch_spec=True)


def window_flops(n_samples, input_dim=64, layers=(3, 4, 6, 3), filters=(32, 64, 128, 256), proj=512, n_fft=512, hop=160):
    """Multiply-adds x 2 of the convs and linears (mel projection included) for one window of n_samples."""
    t, h = n_samples // hop + 1, input_dim
    f = 2 * (n_fft // 2 + 1) * input_dim * t + 2 * 9 * 1 * filters[0] * h * t
    cin = filters[0]
    for s in range(4):
        for i in range(layers[s]):
            if s > 0 and i == 0:
                t, h = (t + 1) // 2, (h + 1) // 2
                f += 2 * cin * filters[s] * h * t                      # downsample 1x1
            f += 2 * 9 * cin * filters[s] * h * t + 2 * 9 * filters[s] * filters[s] * h * t
            f += 2 * 2 * filters[s] * (filters[s] // 8)                 # SE MLP
            cin = filters[s]
    ca = filters[3] * (input_dim // 8)
    return f + 2 * 2 * ca * 128 * t + 2 * 2 * ca * proj


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu-clips", type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    rng = np.random.default_rng(0)
    g = torch.Generator().manual_seed(0)
    clips = [torch.randn(int(rng.uniform(1.5, 8.0) * 16000), generator=g) * 0.1 for _ in range(args.clips)]
    m = ResNetSpeakerEncoder(**KW, audio_config=AUDIO).eval()
    sd = EO.random_state(m.state_dict(), 0)
    m.load_state_dict(sd)
    m.cuda()
    dev = [c.cuda() for c in clips]
    flops = 0
    for c in clips:
        nf = min(c.numel(), 250 * 160)
        flops += 10 * window_flops(nf)

    for _ in range(args.warmup):
        emb = m.compute_embeddings(dev)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        emb = m.compute_embeddings(dev)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps

    # bar: torch eager on the GPU (cuDNN, TF32 off), same clips, one compute_embedding per clip
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sdg = {k: v.cuda() for k, v in sd.items()}

    def eager_all():
        return torch.cat([EO.compute_embedding(sdg, c.unsqueeze(0), AUDIO, **KW) for c in dev])

    with torch.no_grad():
        ref = eager_all()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(max(1, args.steps // 2)):
            eager_all()
        e1.record()
        torch.cuda.synchronize()
    ms_eager = e0.elapsed_time(e1) / max(1, args.steps // 2)
    rel = float((emb.double() - ref.double()).norm(dim=1).max() / ref.double().norm(dim=1).min())

    # bar: torch on the CPU, every host thread
    threads = os.cpu_count()
    torch.set_num_threads(threads)
    n_cpu = min(args.cpu_clips, len(clips))
    with torch.no_grad():
        t0 = time.perf_counter()
        for c in clips[:n_cpu]:
            EO.compute_embedding(sd, c.unsqueeze(0), AUDIO, **KW)
        s_cpu = (time.perf_counter() - t0) / n_cpu

    name, power = card()
    res = {
        "workload": f"{args.clips} clips of 1.5-8 s at 16 kHz, 10 x 250-frame windows each",
        "clips_per_s": round(args.clips / (ms / 1e3), 1),
        "ms_per_batch": round(ms, 2),
        "tflops": round(flops / (ms / 1e3) / 1e12, 2),
        "gflop_per_clip": round(flops / args.clips / 1e9, 2),
        "eager_gpu_clips_per_s": round(args.clips / (ms_eager / 1e3), 1),
        "cpu_clips_per_s": round(1.0 / s_cpu, 2),
        "cpu_threads": threads,
        "parity": rel <= 1e-4,
        "max_rel_err_vs_eager": rel,
        "gpu": name,
        "power_limit": power,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
