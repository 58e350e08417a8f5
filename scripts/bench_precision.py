#!/usr/bin/env python
"""Decoder precision benchmark: the cfg2 batch of bench.py (32 utterances x 64 tokens, same model, tokens and noise)
through Vits.inference with the decoder's tensor-core convs in fp32 (the split-fp16 default), bf16 and fp16 (add
tf32x3 to --precisions for 3xTF32).  Prints one JSON line.

  python scripts/bench_precision.py [--steps K] [--precisions fp32,bf16,fp16]

The precisions are timed alternately, step by step (a 256 MiB L2-evicting write before each timed call, outside the
events).  Per precision: ms per step and M samples/s (valid samples, as bench.py counts them), the decoder stage time
(CUDA events around Vits' waveform_decoder stage), and the waveform's relative RMS error against the fp32 decoder on the
valid samples of the same inputs.  The card's name and power limit are part of the line."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402  (the headline workload's model and batch)
from bench_stream import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--precisions", default="fp32,bf16,fp16")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_precision.py needs a CUDA device: there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    precisions = args.precisions.split(",")
    models = {}
    for p in precisions:                                           # same seed: identical weights, one packing each
        models[p] = bench.build_model().to(dev)
        models[p].trim_padding = not os.environ.get("BENCH_DENSE")
        models[p].waveform_decoder.precision = p
    tokens, lengths, sdp_noise = (t.to(dev) for t in bench.make_batch(0))
    aux = {"x_lengths": lengths}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def prior_noise(shape):
        return torch.randn(shape, generator=torch.Generator(device=dev).manual_seed(99), device=dev, dtype=torch.float32)

    def run(p, events=None):
        model = models[p]
        model._stage_events = events
        try:
            return model.inference(tokens, aux, sdp_noise=sdp_noise, prior_noise=prior_noise, return_alignments=False)
        finally:
            model._stage_events = None

    ref = run("fp32" if "fp32" in models else precisions[0])
    ref_wav = ref["model_outputs"]
    valid = torch.arange(ref_wav.shape[-1], device=dev)[None, None, :] < ref["wav_lengths"][:, None, None]
    samples = int(ref["wav_lengths"].sum())
    line = {"metric": "cfg2_decoder_precision", "card": card(0), "steps": args.steps,
            "batch": f"{bench.B_PER_GPU} x {bench.T_TEXT} tokens", "frames": int(ref["y_mask"].shape[-1]),
            "samples_per_step": samples,
            "padding": "ragged (Vits.trim_padding)" if models[precisions[0]].trim_padding else "dense"}
    err = {}
    for p in precisions:                                           # warm-up, and the error pass
        for _ in range(2):
            w = run(p)["model_outputs"]
        e = (w - ref_wav)[valid].double()
        err[p] = {"rel_rms_vs_fp32": float(e.pow(2).mean().sqrt() / ref_wav[valid].double().pow(2).mean().sqrt()),
                  "finite": bool(torch.isfinite(w).all())}
    step_ms = {p: [] for p in precisions}
    dec_ms = {p: [] for p in precisions}
    for _ in range(args.steps):
        for p in precisions:                                       # alternating, step by step
            flush.fill_(1)
            torch.cuda.synchronize()
            stage = []
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            run(p, stage)
            e.record()
            torch.cuda.synchronize()
            step_ms[p].append(s.elapsed_time(e))
            dec_ms[p].append(sum(a.elapsed_time(b) for n, a, b in stage if n == "waveform_decoder"))
    for p in precisions:
        m = statistics.mean(step_ms[p])
        line[p] = {"ms_per_step": m, "ms_per_step_min_max": [min(step_ms[p]), max(step_ms[p])],
                   "M_samples_per_s": samples / m / 1e3, "decoder_ms": statistics.mean(dec_ms[p]),
                   "decoder_ms_min_max": [min(dec_ms[p]), max(dec_ms[p])], **err[p]}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
