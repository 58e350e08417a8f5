#!/usr/bin/env python
"""Tacotron2 inference on the GPU: Tacotron2Config at its defaults plus double_decoder_consistency (r = 2) with seeded
test weights (tests/tacotron2_oracle.py seeded_weights), 32 utterances of 40-64 tokens, the stop held off (stopnet bias
-30) so every row runs a fixed number of decoder steps (--steps, default 200).

Reports: ms per call and per decoder step for ``inference`` at B = 32 and at B = 1 (CUDA events around whole calls
after warm-up), mel frames/s, the counted weight bytes per step and the HBM time they bound (derived from the data
sheet's 3.35 TB/s, not measured), the Tacotron2 -> vocoder_input -> HiFiGAN v2-shaped generator chain, and the fp32
oracle in torch eager one row at a time (as the reference runs) on the same GPU for the first rows.  The card's name
and power limit are read in the same run.  Prints one JSON line.

--profile: instead, one B = 32 call under torch.profiler (CUDA activity, a run of its own): device time per kernel
name, summed, with launch counts, and the call's total kernel time."""
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

import tacotron2_oracle as TO  # noqa: E402
from ref_golden import layout, seeded_state_dict  # noqa: E402
from tts_b200 import tacotron2 as TC  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def timed(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def weight_bytes_per_step(sd, r_init, c):
    """FP32 weights a decoder step reads: prenet, both LSTMCells, the attention's query layer, projection, stopnet."""
    keys = ["decoder.prenet.linear_layers.0.linear_layer.weight", "decoder.prenet.linear_layers.1.linear_layer.weight",
            "decoder.attention_rnn.weight_ih", "decoder.attention_rnn.weight_hh", "decoder.decoder_rnn.weight_ih",
            "decoder.decoder_rnn.weight_hh", "decoder.attention.query_layer.linear_layer.weight",
            "decoder.linear_projection.linear_layer.weight", "decoder.stopnet.1.linear_layer.weight"]
    return 4 * sum(sd[k].numel() for k in keys)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--eager-rows", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tacotron2 needs a GPU"
    dev = torch.device("cuda:0")
    cfg = TC.Tacotron2Config(num_chars=40, double_decoder_consistency=True, max_decoder_steps=args.steps)
    model = TC.Tacotron2(cfg)
    sd = TO.seeded_weights(seeded_state_dict(layout(model.state_dict()), 13), 17, stop_bias=-30.0)
    model.load_state_dict(sd)
    model.eval().to(dev)
    g = torch.Generator().manual_seed(9)
    lens = torch.randint(40, 65, (32,), generator=g)
    text = torch.zeros(32, int(lens.max()), dtype=torch.long)
    for b, n in enumerate(lens.tolist()):
        text[b, :n] = torch.randint(1, 40, (n,), generator=g)
    text_d, aux = text.to(dev), {"x_lengths": lens.to(dev)}
    res = {"card": card(), "batch": 32, "decoder_steps": args.steps, "r": cfg.r}
    for _ in range(args.warmup):
        out = model.inference(text_d, aux)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model.inference(text_d, aux)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                k = kern.setdefault(ev.name, [0.0, 0])
                k[0] += ev.device_time_total / 1e3
                k[1] += 1
        total = sum(v[0] for v in kern.values())
        top = sorted(kern.items(), key=lambda kv: -kv[1][0])[:12]
        res["profile_total_kernel_ms"] = total
        res["profile_kernels"] = [{"name": n[:90], "ms": round(v[0], 3), "launches": v[1],
                                   "us_per_launch": round(1e3 * v[0] / max(v[1], 1), 2)} for n, v in top]
        print(json.dumps(res))
        return
    assert out["model_outputs_len"].tolist() == [args.steps * cfg.r] * 32
    ms = timed(lambda: model.inference(text_d, aux), args.reps)
    res["ms_per_call_b32"] = ms
    res["us_per_step_b32"] = 1e3 * ms / args.steps
    res["mel_frames_per_s_b32"] = 32 * args.steps * cfg.r / (ms / 1e3)
    one, one_aux = text_d[:1, :int(lens[0])], {"x_lengths": lens[:1].to(dev)}
    model.inference(one, one_aux)
    ms1 = timed(lambda: model.inference(one, one_aux), args.reps)
    res["ms_per_call_b1"] = ms1
    res["us_per_step_b1"] = 1e3 * ms1 / args.steps
    res["step_ratio_b32_over_b1"] = ms / ms1
    wb = weight_bytes_per_step(sd, cfg.r, cfg.out_channels)
    res["weight_mb_per_step"] = wb / 1e6
    res["hbm_bound_us_per_step_derived"] = 1e6 * wb / HBM_BYTES_PER_S
    res["share_of_hbm_bound_b32"] = res["hbm_bound_us_per_step_derived"] / res["us_per_step_b32"]
    # chain into a HiFiGAN v2-shaped generator
    from tts_b200.hifigan import HifiganGenerator
    from tts_b200.vocoder import AudioNorm, vocoder_input
    norm = AudioNorm(signal_norm=True, symmetric_norm=True, max_norm=4.0, clip_norm=True, min_level_db=-100.0,
                     ref_level_db=20.0)
    gen = HifiganGenerator(in_channels=80, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
                           resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4],
                           upsample_initial_channel=128, upsample_factors=[8, 8, 2, 2], inference_padding=0,
                           cond_channels=0, conv_pre_weight_norm=False, conv_post_weight_norm=False,
                           conv_post_bias=False).eval().to(dev)

    def chain():
        mel = model.inference(text_d, aux)["model_outputs"]
        return gen(vocoder_input(mel, norm, norm, padding=0, time_last=False))

    chain()
    res["ms_chain_hifigan_v2_b32"] = timed(chain, args.reps)
    # the fp32 oracle in torch eager, one row at a time as the reference runs, on the same GPU
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    n = args.eager_rows

    def eager():
        for b in range(n):
            TO.inference(sd_dev, text_d[b:b + 1, :int(lens[b])], lens[b:b + 1], cfg)

    eager()
    ms_e = timed(eager, 1) / n
    res["ms_eager_per_row_gpu"] = ms_e
    res["ms_eager_b32_extrapolated"] = 32 * ms_e
    res["speedup_vs_eager_one_row_at_a_time"] = 32 * ms_e / ms
    print(json.dumps(res))


if __name__ == "__main__":
    main()
