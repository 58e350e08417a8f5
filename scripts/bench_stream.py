#!/usr/bin/env python
"""Streaming benchmark: the cfg2 batch of bench.py (32 utterances x 64 tokens, same model, tokens and noise) through
Vits.inference_stream, for several chunk sizes.  Prints one JSON line.

  python scripts/bench_stream.py [--steps K] [--chunks 16,32,64]

Per chunk size: time to the first chunk (CUDA events at the call's start and right after the first chunk's conv_post),
the whole streamed call, and the one-shot Vits.inference on the same inputs, timed alternately with it (a 256 MiB
L2-evicting write before each timed call, outside the events); overhead = streamed / one-shot - 1; `parity`: the
concatenated chunks torch.equal the one-shot waveform.  The card's name and power limit are part of the line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the headline workload's model and batch)


def card(index):
    import torch
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "sm_max_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        p, c = (v.strip() for v in q.strip().split(",")[:2])
        info["power_limit_w"], info["sm_max_mhz"] = float(p), float(c)
    except Exception:  # noqa: BLE001 - the numbers stand without it, labelled unknown
        pass
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--chunks", default="16,32,64")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_stream.py needs a CUDA device: there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = bench.build_model().to(dev)
    model.trim_padding = not os.environ.get("BENCH_DENSE")
    tokens, lengths, sdp_noise = (t.to(dev) for t in bench.make_batch(0))
    aux = {"x_lengths": lengths}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def prior_noise(shape):
        return torch.randn(shape, generator=torch.Generator(device=dev).manual_seed(99), device=dev, dtype=torch.float32)

    def one_shot(ev=None):
        if ev:
            ev[0].record()
        out = model.inference(tokens, aux, sdp_noise=sdp_noise, prior_noise=prior_noise, return_alignments=False)
        if ev:
            ev[1].record()
        return out

    def streamed(chunk, ev=None):
        chunks = []
        if ev:
            ev[0].record()
        for i, c in enumerate(model.inference_stream(tokens, aux, chunk_frames=chunk, sdp_noise=sdp_noise,
                                                     prior_noise=prior_noise)):
            if i == 0 and ev:
                ev[1].record()
            chunks.append(c["model_outputs"])
        if ev:
            ev[2].record()
        return chunks

    def timed(fn, n_ev):
        flush.fill_(1)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(n_ev)]
        fn(ev)
        torch.cuda.synchronize()
        return [ev[0].elapsed_time(e) for e in ev[1:]]

    want = one_shot()["model_outputs"]
    line = {"metric": "cfg2_stream", "card": card(0), "steps": args.steps,
            "batch": f"{bench.B_PER_GPU} x {bench.T_TEXT} tokens", "frames": int(want.shape[-1]) // 256,
            "padding": "ragged windows (Vits.trim_padding)" if model.trim_padding else "dense"}
    for chunk in (int(c) for c in args.chunks.split(",")):
        chunks = streamed(chunk)                                   # warm-up, and the parity pass
        parity = bool(torch.equal(torch.cat(chunks, dim=-1), want))
        first, total, whole = [], [], []
        for _ in range(args.steps):
            f, t = timed(lambda ev: streamed(chunk, ev), 3)
            first.append(f)
            total.append(t)
            whole.append(timed(one_shot, 2)[0])
        m_total, m_whole = statistics.mean(total), statistics.mean(whole)
        line[f"chunk_frames_{chunk}"] = {
            "chunks": len(chunks), "first_chunk_ms": statistics.mean(first), "total_ms": m_total,
            "one_shot_ms": m_whole, "overhead": m_total / m_whole - 1.0, "parity": parity,
            "first_chunk_ms_min_max": [min(first), max(first)], "total_ms_min_max": [min(total), max(total)],
            "one_shot_ms_min_max": [min(whole), max(whole)]}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
