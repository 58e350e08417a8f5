"""ForwardTTS (FastPitch) throughput: default FastPitchConfig, 32 utterances of 40-64 tokens, seeded weights with the
duration predictor's output bias at log 6 (5 frames per token).

Times (a) the batched drop-in ``ForwardTTS.inference`` on the whole batch, (b) the drop-in one utterance at a time,
(c) the CPU oracle (tests/forward_tts_oracle.py) in torch eager on the GPU, one utterance at a time with TF32 off (the
way the reference can run: its inference does not batch), and (d) the oracle on the host CPU with its thread count.
Then the chain of the batched call into a HiFiGAN v2-shaped generator (upsample_initial_channel 128, hop 256), and the
share of the attention kernel in one long utterance (>= 2000 frames), from torch.profiler's CUDA kernel times.  Prints
the parity of the batched call against the eager run, the card's name and its power limit, then one JSON line.

    python scripts/bench_forward_tts.py [--steps 10] [--warmup 3] [--cpu-steps 1]
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
import forward_tts_oracle as FO  # noqa: E402
from ref_golden import layout, seeded_state_dict  # noqa: E402
from tts_b200.forward_tts import FastPitchConfig, ForwardTTS, ForwardTTSArgs  # noqa: E402
from tts_b200.vocoder import GAN, AudioNorm, HifiganConfig, vocoder_input  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def state(model, seed):
    """Seeded weights (LayerNorm gains about 1, the real positional encoding), duration-predictor bias log 6."""
    sd = seeded_state_dict(layout(model.state_dict()), seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in sd:
        if (".norm1." in k or ".norm2." in k) and k.endswith("weight"):
            sd[k] = 1.0 + 0.05 * torch.randn(sd[k].shape, generator=g)
    sd["pos_encoder.pe"] = model.pos_encoder.pe.clone()
    sd["duration_predictor.proj.bias"] = torch.full((1,), math.log(6.0))
    return sd


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, out


def attention_share(m, dev, tokens=420):
    """Kernel time of the decoder attention over all kernel time of one utterance of tokens * 5 frames."""
    x = torch.randint(0, 100, (1, tokens), generator=torch.Generator().manual_seed(5)).to(dev)
    for _ in range(2):
        out = m.inference(x, {})
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            m.inference(x, {})
        torch.cuda.synchronize()
    total = attn = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if ev.key.startswith("Memcpy") or ev.key.startswith("Memset") or t <= 0:
            continue
        total += t
        if "attention_tc3_kernel" in ev.key:
            attn += t
    return int(out["y_lengths"][0]), attn / 3 / 1e3, total / 3 / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-steps", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    dev = torch.device("cuda:0")
    cfg = FastPitchConfig(model_args=ForwardTTSArgs(num_chars=100))
    m = ForwardTTS(cfg).eval()
    sd = state(m, 21)
    m.load_state_dict(sd)
    m.to(dev)
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(40, 65, (32,), generator=g)
    lens[0] = 64
    x = torch.randint(0, 100, (32, 64), generator=g)
    xd, aux = x.to(dev), {"x_lengths": lens.to(dev)}
    rows = [xd[i: i + 1, : int(lens[i])] for i in range(32)]
    torch.manual_seed(3)
    hc = HifiganConfig()
    hc.generator_model_params["upsample_initial_channel"] = 128
    gan = GAN(hc).eval().to(dev)

    def batched():
        return m.inference(xd, aux)

    def one_by_one():
        return [m.inference(r, {}) for r in rows]

    def chain():
        mel = m.inference(xd, aux)["model_outputs"]
        v = vocoder_input(mel, AudioNorm.identity(), AudioNorm.identity(), padding=5, time_last=False, aligned=True)
        return gan.model_g(v)

    for _ in range(args.warmup):
        batched()
        one_by_one()
        chain()
    ms_batched, out = timed(batched, args.steps)
    ms_rows, _ = timed(one_by_one, max(1, args.steps // 2))
    ms_chain, wav = timed(chain, args.steps)
    frames = int(out["y_lengths"].sum())

    # bar: the oracle in torch eager on the same GPU, one utterance at a time, TF32 off
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sdg = {k: v.to(dev) for k, v in sd.items()}
    a = cfg.model_args
    with torch.no_grad():
        def eager_rows():
            return [FO.inference_one(sdg, r, a) for r in rows]

        ref = eager_rows()
        ms_eager, _ = timed(eager_rows, max(1, args.steps // 2))
    same_len = all(int(out["y_lengths"][i]) == int(ref[i]["y_lengths"][0]) for i in range(32))
    err = 0.0
    if same_len:
        num = den = 0.0
        for i in range(32):
            n = int(out["y_lengths"][i])
            d = out["model_outputs"][i, :n] - ref[i]["model_outputs"][0]
            num += float(d.pow(2).sum())
            den += float(ref[i]["model_outputs"][0].pow(2).sum())
        err = math.sqrt(num / den)
    else:
        err = float("inf")

    # bar: the oracle on the host CPU, one utterance at a time
    threads = torch.get_num_threads()
    with torch.no_grad():
        t0 = time.perf_counter()
        for _ in range(args.cpu_steps):
            for i in range(32):
                FO.inference_one(sd, x[i: i + 1, : int(lens[i])], a)
        s_cpu = (time.perf_counter() - t0) / args.cpu_steps

    long_frames, attn_ms, kern_ms = attention_share(m, dev)
    name, power = card()
    print(f"parity: y_lengths equal {same_len}, model_outputs relative RMS error vs eager {err:.2e}")
    print(f"card: {name}, power limit {power}")
    res = {
        "workload": "FastPitch default config, 32 x 64 tokens (40-64 valid), 5 frames/token; chain: + HiFiGAN "
                    "v2-shaped generator, hop 256",
        "mel_frames": frames,
        "batched_ms": round(ms_batched, 2),
        "batched_mel_frames_per_s": round(frames / (ms_batched / 1e3)),
        "one_by_one_ms": round(ms_rows, 2),
        "eager_gpu_one_by_one_ms": round(ms_eager, 2),
        "cpu_one_by_one_ms": round(s_cpu * 1e3, 1),
        "cpu_threads": threads,
        "chain_ms": round(ms_chain, 2),
        "chain_audio_samples_per_s": round(frames * 256 / (ms_chain / 1e3)),
        "long_utterance_frames": long_frames,
        "long_attention_kernel_ms": round(attn_ms, 3),
        "long_all_kernels_ms": round(kern_ms, 3),
        "long_attention_share": round(attn_ms / kern_ms, 3) if kern_ms else None,
        "parity": bool(same_len and err <= 1e-4),
        "gpu": name,
        "power_limit": power,
    }
    print(json.dumps(res))
    assert wav.shape[0] == 32


if __name__ == "__main__":
    main()
