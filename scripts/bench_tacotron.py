#!/usr/bin/env python
"""Tacotron (1) inference on the GPU: TacotronConfig at its defaults (r = 2, out_channels 513) plus
double_decoder_consistency with seeded test weights (tests/tacotron_oracle.py seeded_weights), 32 utterances of 40-64
tokens.  The stopnet bias is -30 and max_decoder_steps is --steps - 1, so every row runs exactly --steps decoder steps
(default 200, 400 frames): the cap decides the stop, not the weights.

Reports: ms per ``inference`` call at B = 32 and at B = 1 (CUDA events around whole calls after warm-up), µs per decoder
step, the split into encoder, loop and postnet (host clock around each library call, each ending in a device
synchronise), the persistent biGRU kernel's time per step (torch.profiler, a run of its own), the fp32 oracle in torch
eager one row at a time (as the reference runs) on the same GPU for the first rows, and the GPU output's relative RMS
difference from that eager run.  The card's name and power limit are read in the same run.  Prints one JSON line."""
import argparse
import ctypes
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

import tacotron_oracle as TO  # noqa: E402
from ref_golden import layout, seeded_state_dict  # noqa: E402
from tts_b200 import _lib  # noqa: E402
from tts_b200 import tacotron as TC  # noqa: E402


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


def split(model, text, lens, steps, reps):
    """ms of the encode, decode_loop and postnet library calls of one B-row inference, as inference() makes them."""
    dev, (b, tt), r, c = text.device, text.shape, model.decoder.r, model.decoder_output_dim
    f32 = dict(dtype=torch.float32, device=dev)
    enc, dec = torch.empty((b, tt, 256), **f32), torch.empty((b, steps * r, c), **f32)
    stop, align = torch.empty((b, steps), **f32), torch.empty((b, steps, tt), **f32)
    out = torch.empty((b, steps * r, model.out_channels), **f32)
    frames = torch.full((b,), steps * r, dtype=torch.int32, device=dev)
    n = (ctypes.c_int32 * b)()
    h, L, s = model.handle(dev), _lib.lib(), _lib.stream_ptr(dev)
    ws = _lib.workspace(dev, L.b200tts_tacotron_workspace_bytes(h, b, tt, steps * r), "tacotron")
    wsp, wsn = _lib.ptr(ws), ctypes.c_size_t(ws.numel())
    calls = {
        "encoder": lambda: L.b200tts_tacotron_encode(h, _lib.ptr(text), _lib.ptr(lens), b, tt, _lib.ptr(enc), wsp, wsn,
                                                     s),
        "loop": lambda: L.b200tts_tacotron_decode_loop(h, _lib.ptr(lens), _lib.ptr(enc), b, tt, r, steps - 1, None,
                                                       32, _lib.ptr(dec), _lib.ptr(stop), _lib.ptr(align), n, wsp,
                                                       wsn, s),
        "postnet": lambda: L.b200tts_tacotron_postnet(h, _lib.ptr(dec), _lib.ptr(frames), b, steps * r, steps * r,
                                                      _lib.ptr(out), wsp, wsn, s)}
    res = {}
    for name, fn in calls.items():
        fn()   # the loop needs the encoder's state: run in order, then time each
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            _lib.check(fn(), name)
            torch.cuda.synchronize()
        res[name] = 1e3 * (time.perf_counter() - t0) / reps
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--eager-rows", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tacotron needs a GPU"
    dev = torch.device("cuda:0")
    cfg = TC.TacotronConfig(num_chars=40, double_decoder_consistency=True, max_decoder_steps=args.steps - 1)
    model = TC.Tacotron(cfg)
    sd = TO.seeded_weights(seeded_state_dict(layout(model.state_dict()), 13), 17, stop_bias=-30.0)
    model.load_state_dict(sd)
    model.eval().to(dev)
    g = torch.Generator().manual_seed(9)
    lens = torch.randint(40, 65, (32,), generator=g)
    text = torch.zeros(32, int(lens.max()), dtype=torch.long)
    for b, n in enumerate(lens.tolist()):
        text[b, :n] = torch.randint(1, 40, (n,), generator=g)
    text_d, lens_d = text.to(dev), lens.to(dev)
    aux = {"x_lengths": lens_d}
    res = {"card": card(), "batch": 32, "decoder_steps": args.steps, "r": cfg.r, "out_channels": cfg.out_channels}
    for _ in range(args.warmup):
        out = model.inference(text_d, aux)
    assert out["model_outputs_len"].tolist() == [args.steps * cfg.r] * 32, out["model_outputs_len"].tolist()
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model.inference(text_d, aux)
            torch.cuda.synchronize()
        kern = {}
        bigru = []
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                k = kern.setdefault(ev.name, [0.0, 0])
                k[0] += ev.device_time_total / 1e3
                k[1] += 1
                if "bigru_kernel" in ev.name:
                    bigru.append(ev.device_time_total)
        total = sum(v[0] for v in kern.values())
        top = sorted(kern.items(), key=lambda kv: -kv[1][0])[:14]
        res["profile_total_kernel_ms"] = total
        res["profile_kernels"] = [{"name": n[:90], "ms": round(v[0], 3), "launches": v[1],
                                   "us_per_launch": round(1e3 * v[0] / max(v[1], 1), 2)} for n, v in top]
        # the encoder's biGRU runs max(lens) steps at most, the postnet's steps * r (every row the same)
        if len(bigru) == 2:
            res["bigru_us_per_step_encoder"] = bigru[0] / int(lens.max())
            res["bigru_us_per_step_postnet"] = bigru[1] / (args.steps * cfg.r)
        print(json.dumps(res))
        return
    ms = timed(lambda: model.inference(text_d, aux), args.reps)
    res["ms_per_call_b32"] = ms
    res["us_per_step_b32"] = 1e3 * ms / args.steps
    res["frames_per_s_b32"] = 32 * args.steps * cfg.r / (ms / 1e3)
    res["split_ms_b32"] = split(model, text_d, lens_d, args.steps, args.reps)
    res["us_per_decoder_step_b32_loop_only"] = 1e3 * res["split_ms_b32"]["loop"] / args.steps
    one, one_aux = text_d[:1, :int(lens[0])], {"x_lengths": lens_d[:1]}
    model.inference(one, one_aux)
    ms1 = timed(lambda: model.inference(one, one_aux), args.reps)
    res["ms_per_call_b1"] = ms1
    res["us_per_step_b1"] = 1e3 * ms1 / args.steps
    res["split_ms_b1"] = split(model, one.contiguous(), lens_d[:1].contiguous(), args.steps, args.reps)
    res["us_per_decoder_step_b1_loop_only"] = 1e3 * res["split_ms_b1"]["loop"] / args.steps
    # the fp32 oracle in torch eager, one row at a time as the reference runs, on the same GPU
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    n = args.eager_rows
    eager_out = []

    def eager():
        eager_out.clear()
        for b in range(n):
            eager_out.append(TO.inference(sd_dev, text_d[b:b + 1, :int(lens[b])], lens[b:b + 1], cfg))

    eager()
    ms_e = timed(eager, 1) / n
    res["ms_eager_per_row_gpu"] = ms_e
    res["ms_eager_b32_extrapolated"] = 32 * ms_e
    res["speedup_vs_eager_one_row_at_a_time"] = 32 * ms_e / ms
    got = model.inference(text_d, aux)
    for k in ("model_outputs", "decoder_outputs"):
        num = sum(float((got[k][b].double().cpu() - eager_out[b][k][0].double().cpu()).pow(2).sum()) for b in range(n))
        den = sum(float(eager_out[b][k][0].double().cpu().pow(2).sum()) for b in range(n))
        res[f"rel_rms_vs_eager_{k}"] = (num / den) ** 0.5
    print(json.dumps(res))


if __name__ == "__main__":
    main()
