"""MelGAN vocoder throughput on bench_glow_tts.py's batch shape: 32 utterances, about 10k mel frames in all (the
Glow-TTS default config, 32 x 64 tokens, ~5 frames per token), random weights.

Times the multi-band (MultibandMelganConfig: (8, 4, 2), 4 residual blocks, base 384, + PQMF) and full-band
(FullbandMelganConfig: melgan_generator, (8, 8, 2, 2), 4 residual blocks, base 512) generators' ``inference`` alone, in
audio samples/s, and the Glow-TTS -> ``vocoder_input`` -> multi-band MelGAN chain next to the same chain into HiFiGAN v1.
Bars on the same batch: the CPU oracle (tests/melgan_oracle.py) in torch eager on the GPU with TF32 off, and on the host
CPU with the thread count stated.  Prints the parity of the kernels against the eager GPU run, the card's name and its
power limit, then one JSON line.

    python scripts/bench_melgan.py [--steps 10] [--warmup 3] [--cpu-steps 1]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "scripts")):
    sys.path.insert(0, p)
import melgan_oracle as MO  # noqa: E402
from bench_glow_tts import batch, card, timed  # noqa: E402
from ref_golden import layout, seeded_state_dict  # noqa: E402
from tts_b200.glow_tts import GlowTTS  # noqa: E402
from tts_b200.vocoder import (GAN, AudioNorm, FullbandMelganConfig, HifiganConfig, MultibandMelganConfig,  # noqa: E402
                              vocoder_input)


def vocoder(config, seed):
    gan = GAN(config).eval()
    g = gan.model_g
    sd = seeded_state_dict(layout(g.state_dict()), seed)
    for k, v in g.state_dict().items():
        if k.startswith("pqmf_layer."):
            sd[k] = v.clone()
    g.load_state_dict(sd)
    return gan, sd


def oracle_kw(g):
    c = g._cfg
    return dict(upsample_factors=tuple(c["upsample_factors"]), num_res_blocks=c["num_res_blocks"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-steps", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    dev = torch.device("cuda:0")
    cfg, sd, x, lens = batch()
    glow = GlowTTS(cfg).eval()
    glow.load_state_dict(sd)
    glow.to(dev)
    xd, aux = x.to(dev), {"x_lengths": lens.to(dev)}
    with torch.no_grad():
        mel = glow.inference(xd, aux)["model_outputs"]             # [32, T, 80]: the vocoders' input
    mel_bct = mel.transpose(1, 2).contiguous()
    frames = int(mel.shape[0] * mel.shape[1])

    mb, mb_sd = vocoder(MultibandMelganConfig(), 31)
    fb, fb_sd = vocoder(FullbandMelganConfig(), 32)
    torch.manual_seed(3)
    hifi = GAN(HifiganConfig()).eval()
    for m in (mb, fb, hifi):
        m.to(dev)

    def chain(gan, pad):
        def run():
            m = glow.inference(xd, aux)["model_outputs"]
            return gan.inference(m.transpose(1, 2)) if pad == 2 else gan.model_g(
                vocoder_input(m, AudioNorm.identity(), AudioNorm.identity(), padding=pad, time_last=False, aligned=True))
        return run

    runs = {"multiband": lambda: mb.inference(mel_bct), "fullband": lambda: fb.inference(mel_bct),
            "chain_multiband": chain(mb, 2), "chain_hifigan": chain(hifi, 5)}
    for _ in range(args.warmup):
        for f in runs.values():
            f()
    ms, outs = {}, {}
    for k, f in runs.items():
        ms[k], outs[k] = timed(f, args.steps)
    samples = {k: outs[k].shape[0] * outs[k].shape[-1] for k in ("multiband", "fullband")}

    # bar: the oracle in torch eager on the same GPU, TF32 off
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    mbg = {k: v.to(dev) for k, v in mb_sd.items()}
    fbg = {k: v.to(dev) for k, v in fb_sd.items()}
    with torch.no_grad():
        eager = {"multiband": lambda: MO.inference(mbg, mel_bct, pqmf=True, **oracle_kw(mb.model_g)),
                 "fullband": lambda: MO.inference(fbg, mel_bct, **oracle_kw(fb.model_g))}
        ref = {k: f() for k, f in eager.items()}
        ms_eager = {k: timed(f, max(1, args.steps // 2))[0] for k, f in eager.items()}
    err = {k: float((outs[k] - ref[k]).pow(2).mean().sqrt() / ref[k].pow(2).mean().sqrt()) for k in ref}

    # bar: the oracle on the host CPU (multi-band)
    threads = torch.get_num_threads()
    mel_cpu = mel_bct.cpu()
    with torch.no_grad():
        t0 = time.perf_counter()
        for _ in range(args.cpu_steps):
            MO.inference(mb_sd, mel_cpu, pqmf=True, **oracle_kw(mb.model_g))
        s_cpu = (time.perf_counter() - t0) / args.cpu_steps

    name, power = card()
    print("parity: relative RMS error vs eager " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    print(f"card: {name}, power limit {power}")
    res = {
        "workload": "32 utterances, Glow-TTS default mel (~5 frames/token), padded batch; MultibandMelganConfig / "
                    "FullbandMelganConfig generators, random weights",
        "mel_frames": frames,
        "multiband_ms": round(ms["multiband"], 2),
        "multiband_audio_samples_per_s": round(samples["multiband"] / (ms["multiband"] / 1e3)),
        "fullband_ms": round(ms["fullband"], 2),
        "fullband_audio_samples_per_s": round(samples["fullband"] / (ms["fullband"] / 1e3)),
        "chain_multiband_ms": round(ms["chain_multiband"], 2),
        "chain_hifigan_v1_ms": round(ms["chain_hifigan"], 2),
        "eager_gpu_multiband_ms": round(ms_eager["multiband"], 2),
        "eager_gpu_fullband_ms": round(ms_eager["fullband"], 2),
        "cpu_multiband_ms": round(s_cpu * 1e3, 1),
        "cpu_threads": threads,
        "parity": bool(max(err.values()) <= 1e-4),
        "gpu": name,
        "power_limit": power,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
