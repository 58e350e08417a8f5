"""Glow-TTS throughput on bench.py's batch shape: 32 utterances of up to 64 tokens, default GlowTTSConfig, random
weights with the duration predictor's output bias at log 6 (about 5 frames per token, LJSpeech-like).

Times ``GlowTTS.inference`` alone (mel frames/s) and chained through ``vocoder_input`` into a HiFiGAN v1 generator
(80 mel, hop 256: audio samples/s).  Bars on the same batch: the CPU oracle (tests/glow_oracle.py) in torch eager on the
GPU with TF32 off, and on the host CPU with the thread count stated.  Prints the parity of the kernels against the eager
GPU run, the card's name and its power limit, then one JSON line.

    python scripts/bench_glow_tts.py [--steps 10] [--warmup 3] [--cpu-steps 1]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import glow_oracle as GO  # noqa: E402
import vits_oracle as O  # noqa: E402
from ref_golden import layout, seeded_state_dict  # noqa: E402
from tts_b200.glow_tts import GlowTTS, GlowTTSConfig  # noqa: E402
from tts_b200.vocoder import GAN, AudioNorm, HifiganConfig, vocoder_input  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def batch():
    cfg = GlowTTSConfig(num_chars=100)
    sd = seeded_state_dict(layout(GlowTTS(cfg).state_dict()), 21)
    g = torch.Generator().manual_seed(22)
    for n in range(cfg.num_flow_blocks_dec):
        sd[f"decoder.flows.{3 * n + 1}.weight"] = torch.linalg.qr(torch.randn(4, 4, generator=g))[0]
    sd["encoder.duration_predictor.proj.bias"] = torch.full((1,), math.log(6.0))
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(40, 65, (32,), generator=g)
    lens[0] = 64
    x = torch.randint(0, 100, (32, 64), generator=g)
    return cfg, sd, x, lens


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-steps", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    dev = torch.device("cuda:0")
    cfg, sd, x, lens = batch()
    m = GlowTTS(cfg).eval()
    m.load_state_dict(sd)
    m.to(dev)
    torch.manual_seed(3)
    gan = GAN(HifiganConfig()).eval()
    voc_sd = {k: v.clone() for k, v in gan.model_g.state_dict().items()}
    gan.to(dev)
    xd, aux = x.to(dev), {"x_lengths": lens.to(dev)}

    def glow():
        return m.inference(xd, aux)

    def chain():
        mel = m.inference(xd, aux)["model_outputs"]
        v = vocoder_input(mel, AudioNorm.identity(), AudioNorm.identity(), padding=5, time_last=False, aligned=True)
        return gan.model_g(v)

    for _ in range(args.warmup):
        glow()
        chain()
    ms_glow, out = timed(glow, args.steps)
    ms_chain, wav = timed(chain, args.steps)
    frames = int(out["y_lengths"].sum())                     # valid mel frames of the batch
    samples = frames * 256

    # bar: the oracle in torch eager on the same GPU, TF32 off
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sdg = {k: v.to(dev) for k, v in sd.items()}
    voc_g = {k: v.to(dev) for k, v in voc_sd.items()}
    with torch.no_grad():
        def eager_glow():
            return GO.inference(sdg, xd, aux["x_lengths"], cfg)

        def eager_chain():
            mel = GO.inference(sdg, xd, aux["x_lengths"], cfg)["model_outputs"]
            return O.hifigan_inference(voc_g, mel.transpose(1, 2), 5)

        ref = eager_glow()
        eager_chain()
        ms_eager_glow, _ = timed(eager_glow, max(1, args.steps // 2))
        ms_eager_chain, _ = timed(eager_chain, max(1, args.steps // 2))
    same_len = torch.equal(out["y_lengths"].cpu(), ref["y_lengths"].cpu())
    err = float((out["model_outputs"] - ref["model_outputs"]).pow(2).mean().sqrt() /
                ref["model_outputs"].pow(2).mean().sqrt()) if same_len else float("inf")

    # bar: the oracle on the host CPU
    threads = torch.get_num_threads()
    with torch.no_grad():
        t0 = time.perf_counter()
        for _ in range(args.cpu_steps):
            GO.inference(sd, x, lens, cfg)
        s_cpu = (time.perf_counter() - t0) / args.cpu_steps

    name, power = card()
    print(f"parity: y_lengths equal {same_len}, model_outputs relative RMS error vs eager {err:.2e}")
    print(f"card: {name}, power limit {power}")
    res = {
        "workload": "GlowTTS default config, 32 x 64 tokens (40-64 valid), ~5 frames/token; chain: + HiFiGAN v1, hop 256",
        "mel_frames": frames,
        "glow_ms": round(ms_glow, 2),
        "glow_mel_frames_per_s": round(frames / (ms_glow / 1e3)),
        "chain_ms": round(ms_chain, 2),
        "chain_audio_samples_per_s": round(samples / (ms_chain / 1e3)),
        "eager_gpu_glow_ms": round(ms_eager_glow, 2),
        "eager_gpu_chain_ms": round(ms_eager_chain, 2),
        "cpu_glow_ms": round(s_cpu * 1e3, 1),
        "cpu_threads": threads,
        "parity": bool(same_len and err <= 1e-4),
        "gpu": name,
        "power_limit": power,
    }
    print(json.dumps(res))
    assert wav.shape[0] == 32


if __name__ == "__main__":
    main()
