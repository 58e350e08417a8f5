#!/usr/bin/env python
"""Split-fp16 decoder benchmark: bench.py's cfg2 batch (32 utterances x 64 tokens, same model, tokens and noise) through
Vits.inference with the decoder's tensor-core convs as 3xTF32 (precision "tf32x3") and as the split-fp16 product (the
"fp32" default), then every distinct decoder conv shape on its own.  Prints one JSON line.

  python scripts/bench_split16.py [--steps K] [--layer-steps K]

Both builds are timed alternately, step by step, after two warm-up steps each (a 256 MiB L2-evicting write before each
timed call, outside the events): ms per step, valid M samples/s (as bench.py counts them), CUDA-event time per Vits
stage, and the default run's waveform relative RMS against the tf32x3 run on the valid samples.  Per layer (dense, the
whole batch at the stage's padded length, the same alternation): CUDA-event time per launch in each arithmetic, the
algorithmic FLOPs from the shape, and the MMA-bound share -- the time the layer's MMAs need at the data-sheet dense
rate (3 MMAs per algorithmic multiply-add: TF32 495 TFLOP/s for tf32x3, FP16 989 TFLOP/s for the split) over the
measured time.  The card's name, power limit and max SM clock are read in the same run."""
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

BUILDS = ("tf32x3", "fp32")
LAYER_PREC = {"tf32x3": "tf32x3", "fp32": "f16x3"}        # FusedConv1d name of each build's decoder arithmetic
MMA_PEAK = {"tf32x3": 495e12, "fp32": 989e12}              # H100 SXM data sheet, dense; 3 MMAs per multiply-add either way


def decoder_layers(cfg, frames):
    """Distinct (name, kind, cin, cout, k, dil_or_stride, T_in, count) of the decoder's tensor-core convs at `frames`."""
    out = [("conv_pre", "conv", cfg["in_channels"], cfg["upsample_initial_channel"], 7, 1, frames, 1)]
    ch, t = cfg["upsample_initial_channel"], frames
    for s, (u, k) in enumerate(zip(cfg["upsample_factors"], cfg["upsample_kernel_sizes"])):
        out.append((f"ups{s}", "ups", ch, ch // 2, k, u, t, 1))
        ch, t = ch // 2, t * u
        shapes = {}
        for rk, dils in zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]):
            for d in dils:                                     # ResBlock1: convs1 at dilation d, convs2 at 1
                for dd in (d, 1):
                    shapes[(rk, dd)] = shapes.get((rk, dd), 0) + 1
        for (rk, dd), n in sorted(shapes.items()):
            out.append((f"s{s}_k{rk}_d{dd}", "conv", ch, ch, rk, dd, t, n))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--layer-steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_split16.py needs a CUDA device: there is no CPU fallback"
    from tts_b200.conv import FusedConv1d
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    models = {}
    for p in BUILDS:                                           # same seed: identical weights, one packing each
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

    line = {"metric": "cfg2_decoder_split16", "card": card(0), "steps": args.steps,
            "batch": f"{bench.B_PER_GPU} x {bench.T_TEXT} tokens",
            "padding": "ragged (Vits.trim_padding)" if models[BUILDS[0]].trim_padding else "dense"}
    outs = {}
    for p in BUILDS:                                           # warm-up, and the error pass
        for _ in range(2):
            outs[p] = run(p)
    ref = outs["tf32x3"]
    ref_wav, wav = ref["model_outputs"], outs["fp32"]["model_outputs"]
    valid = torch.arange(ref_wav.shape[-1], device=dev)[None, None, :] < ref["wav_lengths"][:, None, None]
    samples = int(ref["wav_lengths"].sum())
    frames = int(ref["y_mask"].shape[-1])
    e = (wav - ref_wav)[valid].double()
    line.update(frames=frames, samples_per_step=samples,
                wav_rel_rms_fp32_vs_tf32x3=float(e.pow(2).mean().sqrt() / ref_wav[valid].double().pow(2).mean().sqrt()),
                durations_equal=bool(torch.equal(outs["fp32"]["durations"], ref["durations"])),
                finite=bool(torch.isfinite(wav).all()))
    step_ms = {p: [] for p in BUILDS}
    stage_ms = {p: {} for p in BUILDS}
    for _ in range(args.steps):
        for p in BUILDS:                                       # alternating, step by step
            flush.fill_(1)
            torch.cuda.synchronize()
            stage = []
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            run(p, stage)
            e.record()
            torch.cuda.synchronize()
            step_ms[p].append(s.elapsed_time(e))
            for n, a, b in stage:
                stage_ms[p].setdefault(n, []).append(a.elapsed_time(b))
    for p in BUILDS:
        m = statistics.median(step_ms[p])
        line[p] = {"ms_per_step_median": m, "ms_per_step_min_max": [min(step_ms[p]), max(step_ms[p])],
                   "M_samples_per_s": samples / m / 1e3,
                   "stage_ms_median": {n: statistics.median(v) for n, v in stage_ms[p].items()}}

    # ---------------- per layer, dense, whole batch
    cfg = models["fp32"].waveform_decoder._cfg
    layers = []
    b = bench.B_PER_GPU
    gen = torch.Generator().manual_seed(5)
    total = {p: 0.0 for p in BUILDS}
    for name, kind, cin, cout, k, ds, tin, count in decoder_layers(cfg, frames):
        x = torch.randn(b, cin, tin, generator=gen).to(dev)
        if kind == "ups":
            w = torch.randn(cin, cout, k, generator=gen) / (cin * k / ds) ** 0.5
            convs = {p: FusedConv1d(w, torch.zeros(cout), padding=(k - ds) // 2, transposed=True, stride=ds,
                                    precision=LAYER_PREC[p]) for p in BUILDS}
            flop = 2.0 * b * tin * cin * cout * k                  # every input sample meets all k taps of each output channel
        else:
            w = torch.randn(cout, cin, k, generator=gen) / (cin * k) ** 0.5
            convs = {p: FusedConv1d(w, torch.zeros(cout), dilation=ds, padding=(k * ds - ds) // 2,
                                    precision=LAYER_PREC[p]) for p in BUILDS}
            flop = 2.0 * b * tin * cin * cout * k
        for p in BUILDS:
            convs[p](x, in_slope=0.1)
        ms = {p: [] for p in BUILDS}
        for _ in range(args.layer_steps):
            for p in BUILDS:
                flush.fill_(1)
                torch.cuda.synchronize()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                convs[p](x, in_slope=0.1)
                e.record()
                torch.cuda.synchronize()
                ms[p].append(s.elapsed_time(e))
        row = {"layer": name, "cin": cin, "cout": cout, "k": k, ("stride" if kind == "ups" else "dil"): ds, "t_in": tin,
               "count": count, "gflop": flop / 1e9}
        for p in BUILDS:
            med = statistics.median(ms[p])
            total[p] += med * count
            row[p] = {"ms": med, "ms_min_max": [min(ms[p]), max(ms[p])], "tflops": flop / (med / 1e3) / 1e12,
                      "mma_bound_share": (3 * flop / MMA_PEAK[p]) / (med / 1e3)}
        layers.append(row)
        del convs, x
    line["layers"] = layers
    line["layers_sum_ms"] = total                          # counted per occurrence, dense (no ragged skipping)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
