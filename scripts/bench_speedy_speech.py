"""SpeedySpeech throughput: default SpeedySpeechConfig, 32 utterances of 40-64 tokens, seeded weights (BatchNorm
statistics as in tests/test_speedy_speech_oracle_cpu.py) with the duration predictor's output bias at log 6 (5 frames
per token).

Times (a) the batched drop-in ``ForwardTTS.inference`` on the whole batch, (b) the drop-in one utterance at a time,
(c) the CPU oracle (tests/speedy_speech_oracle.py) in torch eager on the GPU, one utterance at a time with TF32 off (the
way the reference can run: its inference does not batch), and (d) the oracle on the host CPU with its thread count.
Then the chain of the batched call into a HiFiGAN v2-shaped generator (upsample_initial_channel 128, hop 256; SpeedySpeech's
default vocoder is hifigan_v2), and the decoder's achieved FLOP/s: 2 x its conv weights x the batch's frames over the
time of its tensor-core conv kernels in torch.profiler's CUDA kernel times (every decoder conv runs on them, no encoder
conv does).  Prints the parity of the batched call against the eager run, the card's name and its power limit, then one
JSON line.

    python scripts/bench_speedy_speech.py [--steps 10] [--warmup 3] [--cpu-steps 1]
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
import speedy_speech_oracle as SO  # noqa: E402
from test_speedy_speech_oracle_cpu import speedy_state  # noqa: E402
from tts_b200.forward_tts import SpeedySpeech, SpeedySpeechConfig  # noqa: E402
from tts_b200.vocoder import GAN, AudioNorm, HifiganConfig, vocoder_input  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, out


def busy_ms(spans):
    """Length of the union of [start, end) intervals (us) in ms: the tensor-core convs start early under programmatic
    stream serialization and wait for their predecessor, so kernel spans overlap and their sum overstates the time."""
    total, end = 0.0, float("-inf")
    for s, e in sorted(spans):
        if e > end:
            total += e - max(s, end)
            end = e
    return total / 1e3


def decoder_kernel_ms(m, xd, aux, calls=3):
    """Per-call GPU time covered by the tensor-core conv kernels (the decoder's convs) and by all kernels, from
    torch.profiler's CUDA kernel events."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            m.inference(xd, aux)
        torch.cuda.synchronize()
    dec, every = [], []
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.key.startswith(("Memcpy", "Memset")):
            continue
        span = (ev.time_range.start, ev.time_range.end)
        every.append(span)
        if "conv1d_tc3" in ev.key:
            dec.append(span)
    return busy_ms(dec) / calls, busy_ms(every) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-steps", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    dev = torch.device("cuda:0")
    cfg = SpeedySpeechConfig()
    cfg.model_args.num_chars = 100
    m = SpeedySpeech(cfg).eval()
    sd = speedy_state(m, 21, 5)
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
            return [SO.inference_one(sdg, r, a) for r in rows]

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
                SO.inference_one(sd, x[i: i + 1, : int(lens[i])], a)
        s_cpu = (time.perf_counter() - t0) / args.cpu_steps

    dec_ms, kern_ms = decoder_kernel_ms(m, xd, aux)
    dec_weights = sum(v.numel() for k, v in m.state_dict().items() if k.startswith("decoder.") and v.dim() == 3)
    dec_flop = 2.0 * dec_weights * frames
    name, power = card()
    print(f"parity: y_lengths equal {same_len}, model_outputs relative RMS error vs eager {err:.2e}")
    print(f"card: {name}, power limit {power}")
    res = {
        "workload": "SpeedySpeech default config, 32 x 64 tokens (40-64 valid), 5 frames/token; chain: + HiFiGAN "
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
        "decoder_gflop": round(dec_flop / 1e9, 2),
        "decoder_conv_kernels_ms": round(dec_ms, 3),
        "decoder_tflop_per_s": round(dec_flop / (dec_ms / 1e3) / 1e12, 2) if dec_ms else None,
        "all_kernels_ms": round(kern_ms, 3),
        "parity": bool(same_len and err <= 1e-4),
        "gpu": name,
        "power_limit": power,
    }
    print(json.dumps(res))
    assert wav.shape[0] == 32


if __name__ == "__main__":
    main()
