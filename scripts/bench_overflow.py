#!/usr/bin/env python
"""Overflow inference on the GPU: the default OverflowConfig with seeded test weights (tests/overflow_oracle.py
seeded_weights), 32 utterances of 40-64 tokens, sampling_temp 0.334.

Reports: ms per batch and mel frames/s for ``inference`` (CUDA events around whole calls after warm-up), the split into
encode / sampling loop / decoder (events between the three C-ABI calls), the loop's time per frame, launches per
frame, the Overflow -> vocoder_input -> HiFiGAN v2-shaped generator chain, and the fp32 oracle in torch eager one row at
a time (as the reference loops) on the same GPU and on the host CPU, for the first rows of the batch.  The card's name
and power limit are read in the same run.  Also reports an upper bound of the per-call cost of building the frame
graph (a one-frame sample() call).  Prints one JSON line."""
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

import overflow_oracle as OO  # noqa: E402
from ref_golden import layout, seeded_state_dict  # noqa: E402
from tts_b200 import _lib  # noqa: E402
from tts_b200 import overflow as OV  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-rows", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_overflow needs a GPU"
    dev = torch.device("cuda:0")
    cfg = OV.OverflowConfig(num_chars=130)
    model = OV.Overflow(cfg)
    sd = OO.seeded_weights(seeded_state_dict(layout(model.state_dict()), 13), 17)
    model.load_state_dict(sd)
    model.eval().to(dev)
    g = torch.Generator().manual_seed(1)
    lens = torch.randint(40, 65, (a.batch,), generator=g)
    text = torch.zeros(a.batch, int(lens.max()), dtype=torch.long)
    for b, n in enumerate(lens.tolist()):
        text[b, :n] = torch.randint(1, 130, (n,), generator=g)
    tx, lx = text.to(dev), lens.to(dev)
    aux = {"x_lengths": lx, "sampling_temp": 0.334}
    torch.manual_seed(0)
    out = model.inference(tx, aux)
    torch.cuda.synchronize()
    frames = out["hmm_outputs_len"].cpu()
    ms = timed(lambda: model.inference(tx, aux), a.reps)

    # the three stages through the C ABI, with events in between
    L = _lib.lib()
    h = model.handle(dev)
    b, tt, mt, c = a.batch, text.shape[1], cfg.max_sampling_time, 80
    noise = torch.randn(b, mt, c, device=dev)
    states = torch.empty(b, tt * 2, 512, device=dev)
    hmm = torch.empty(b, mt, c, device=dev)
    st_tr = torch.empty(b, mt + 1, dtype=torch.int32, device=dev)
    fr = (ctypes.c_int32 * b)()
    ws = _lib.workspace(dev, L.b200tts_overflow_workspace_bytes(h, b, tt, mt), "overflow")
    wsp, wsn, s = _lib.ptr(ws), ctypes.c_size_t(ws.numel()), _lib.stream_ptr(dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    split = []
    for _ in range(a.reps):
        ev[0].record()
        _lib.check(L.b200tts_overflow_encode(h, _lib.ptr(tx), _lib.ptr(lx), b, tt, _lib.ptr(states), wsp, wsn, s), "e")
        ev[1].record()
        _lib.check(L.b200tts_overflow_sample(h, _lib.ptr(lx), b, tt, ctypes.c_float(0.334), mt, ctypes.c_float(0.55),
                                             _lib.ptr(noise), None, OV.CHUNK_FRAMES, _lib.ptr(hmm), _lib.ptr(st_tr), fr,
                                             wsp, wsn, s), "s")
        ev[2].record()
        fmax = max(fr)
        fd = torch.tensor(list(fr), dtype=torch.int32, device=dev)
        mel = torch.empty(b, fmax // 2 * 2, c, device=dev)
        _lib.check(L.b200tts_overflow_decode(h, _lib.ptr(hmm), _lib.ptr(fd), b, fmax, mt, _lib.ptr(mel), wsp, wsn, s),
                   "d")
        ev[3].record()
        torch.cuda.synchronize()
        split.append((ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3]), max(fr)))
    split.sort(key=lambda x: x[1])
    # sample() captures and instantiates its frame graph (32 frames x 6 kernels) on every call: a max_sampling_time = 1
    # call is that set-up plus one replay in which only the first frame does work -- an upper bound of the set-up cost
    setup = []
    for _ in range(a.reps):
        ev[1].record()
        _lib.check(L.b200tts_overflow_sample(h, _lib.ptr(lx), b, tt, ctypes.c_float(0.334), 1, ctypes.c_float(0.55),
                                             _lib.ptr(noise), None, OV.CHUNK_FRAMES, _lib.ptr(hmm), _lib.ptr(st_tr), fr,
                                             wsp, wsn, s), "s1")
        ev[2].record()
        torch.cuda.synchronize()
        setup.append(ev[1].elapsed_time(ev[2]))
    setup.sort()
    setup_ms = setup[len(setup) // 2]
    enc_ms, loop_ms, dec_ms, loop_frames = split[len(split) // 2]
    with _lib.dispatch_log() as log:
        model.inference(tx, aux)
    per_frame = sum(1 for n in log.names if n in ("lstm_cell", "hmm_linear", "hmm_step"))

    # Overflow -> vocoder_input -> HiFiGAN v2-shaped generator
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
        o = model.inference(tx, aux)
        return gen(vocoder_input(o["model_outputs"], norm, norm, padding=0, time_last=False))
    chain()
    chain_ms = timed(chain, a.reps)

    # the oracle, one row at a time, fp32 eager on the GPU and on the host CPU (first rows only)
    rows = list(range(min(a.oracle_rows, a.batch)))
    sd_gpu = {k: v.to(dev) for k, v in sd.items()}

    def oracle_on(sdx, device):
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        t0 = time.perf_counter()
        n = 0
        for r in rows:
            with torch.no_grad():
                enc = OO.encoder(sdx, text[r:r + 1, :int(lens[r])].to(device), cfg)
                x, _, _ = OO.sample(sdx, enc, int(lens[r]) * 2, cfg, 0.334, cfg.max_sampling_time, 0.55)
            n += x.shape[0]
        if device.type == "cuda":
            torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, n

    try:
        oracle_on(sd_gpu, dev)
        og_ms, og_frames = oracle_on(sd_gpu, dev)
    except Exception as e:  # the oracle's meta-device LSTM needs every tensor on one device
        og_ms, og_frames = float("nan"), f"failed: {e}"
    oc_ms, oc_frames = oracle_on(sd, torch.device("cpu"))
    tot = int(frames.sum())
    res = {"workload": f"OverflowConfig defaults, seeded weights, B={a.batch}, tokens 40-64, temp 0.334",
           "card": card(), "inference_ms": round(ms, 2), "mel_frames": tot, "max_frames": int(frames.max()),
           "mel_frames_per_s": round(tot / ms * 1e3), "encode_ms": round(enc_ms, 2), "loop_ms": round(loop_ms, 2),
           "decode_ms": round(dec_ms, 2), "loop_share": round(loop_ms / (enc_ms + loop_ms + dec_ms), 3),
           "loop_frames": loop_frames, "graph_setup_ms_upper_bound": round(setup_ms, 3), "loop_us_per_frame": round(loop_ms / loop_frames * 1e3, 2),
           "launches_per_frame": per_frame, "chain_ms": round(chain_ms, 2),
           "oracle_gpu_eager_ms_per_frame": round(og_ms / og_frames, 3) if isinstance(og_frames, int) else og_frames,
           "oracle_cpu_ms_per_frame": round(oc_ms / oc_frames, 3), "oracle_rows": len(rows)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
