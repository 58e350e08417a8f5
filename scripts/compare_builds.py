#!/usr/bin/env python
"""Outputs and workspace sizes of every engine in this tree against another build of the package, on the same seeded
inputs.

    python scripts/compare_builds.py --other /path/to/other/checkout   (both trees built with __graft_entry__.build())

Runs the same workloads in each tree, each in a subprocess with that tree first on sys.path:
- the autoregressive models on 12 ragged rows of 20-59 tokens with the seeded test weights (tests/overflow_oracle.py,
  tacotron_oracle.py, tacotron2_oracle.py): Overflow at temperature 0, Neural-HMM without prenet dropout, Overflow
  sampled at 0.334 with supplied noise; Tacotron and Tacotron2, each with original + location attention,
  dynamic-convolution attention, the folded "bn" prenet, r below r_init and prenet dropout with supplied draws, and
  Tacotron with a memory queue of 5 frames.  Each records the handle's workspace_bytes for the encoder / loop and for
  the frames it produced;
- every call of tests/test_workspace_gpu.py (the VITS stack, Glow-TTS, FastPitch, the vocoders, the speaker encoder,
  Griffin-Lim, and the autoregressive models at random weights) at B = 1, 3 and two lengths each, seeded, recording
  the workspace sizes the module asks ``_lib.workspace`` for.
Prints one JSON line with ``torch.equal`` per output, ``"equal": true`` when every output matches bit for bit, and the
workspace sizes as [this tree, other tree] per workload.  Writes only to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, MAX_STEPS = 12, 40


def run(tree, out):
    import torch

    sys.path[:0] = [tree, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]   # the tests are this tree's
    import overflow_oracle as OO
    import tacotron2_oracle as T2O
    import tacotron_oracle as T1O
    from ref_golden import layout, seeded_state_dict
    from tts_b200 import _lib
    from tts_b200 import overflow as OV
    from tts_b200 import tacotron as T1
    from tts_b200 import tacotron2 as T2

    assert os.path.realpath(OV.__file__).startswith(os.path.realpath(tree)), OV.__file__
    dev = torch.device("cuda:0")
    L = _lib.lib()
    g = torch.Generator().manual_seed(3)
    lens = torch.randint(20, 60, (B,), generator=g)
    text = torch.zeros(B, int(lens.max()), dtype=torch.long)
    for b, n in enumerate(lens.tolist()):
        text[b, :n] = torch.randint(1, 40, (n,), generator=g)
    tt = text.shape[1]
    res = {}

    def record(kind, m, o, prefix, frames):
        res[kind] = {k: v.cpu() for k, v in o.items() if torch.is_tensor(v)}
        fn = getattr(L, f"b200tts_{prefix}_workspace_bytes")
        h = m.handle(dev)
        res[kind]["workspace_bytes"] = torch.tensor([fn(h, B, tt, 0), fn(h, B, tt, frames)])

    for kind, over in (("overflow", dict(sampling_temp=0.0)), ("neuralhmm", dict(prenet_dropout_at_inference=False)),
                       ("overflow_sampled", dict(sampling_temp=0.334))):
        cls, ccls = (OV.Overflow, OV.OverflowConfig) if kind.startswith("overflow") else \
            (OV.NeuralhmmTTS, OV.NeuralhmmTTSConfig)
        cfg = ccls(num_chars=40, **over)
        m = cls(cfg)
        m.load_state_dict(OO.seeded_weights(seeded_state_dict(layout(m.state_dict()), 13), 17))
        m.eval().to(dev)
        draws = {"noise": torch.randn(B, cfg.max_sampling_time, 80, generator=g).to(dev)}
        o = m.inference(text.to(dev), {"x_lengths": lens.to(dev)}, draws=draws)
        record(kind, m, o, "overflow", int(o["hmm_outputs_len"].max()))

    variants = {"original_location": {}, "dca": dict(attention_type="dynamic_convolution"),
                "prenet_bn": dict(prenet_type="bn"), "r_below_r_init": dict(r=3),
                "dropout": dict(prenet_dropout_at_inference=True), "memory_size_5": dict(memory_size=5)}
    for name, mod, oracle, ccls, cls in (("tacotron", T1, T1O, T1.TacotronConfig, T1.Tacotron),
                                         ("tacotron2", T2, T2O, T2.Tacotron2Config, T2.Tacotron2)):
        for var, over in variants.items():
            if name == "tacotron2" and var == "memory_size_5":   # Tacotron2's decoder has no memory queue
                continue
            cfg = ccls(num_chars=40, max_decoder_steps=MAX_STEPS, **over)
            m = cls(cfg)
            m.load_state_dict(oracle.seeded_weights(seeded_state_dict(layout(m.state_dict()), 13), 17))
            m.eval().to(dev)
            if var == "r_below_r_init":
                m.decoder.set_r(2)
            draws = {"dropout": (torch.rand(B, MAX_STEPS + 1, 2, 256, generator=g) < 0.5).to(dev)}
            o = m.inference(text.to(dev), {"x_lengths": lens.to(dev)}, draws=draws)
            record(f"{name}.{var}", m, o, name, int(o["model_outputs_len"].max()))
    import test_workspace_gpu as W

    real = _lib.workspace
    for name, make in W.CALLS.items():
        torch.manual_seed(0)   # the same weights in both trees
        call = make()
        t0 = call.__defaults__[0]
        for b in (1, 3):
            for t in (t0, 2 * t0 + 1):
                asked = []

                def workspace(device, nbytes, tag="default"):
                    asked.append(int(nbytes))
                    return real(device, nbytes, tag)
                _lib.workspace = workspace
                outs = W.seeded(lambda bb: call(bb, t), b)
                _lib.workspace = real
                res[f"{name}.B{b}.T{t}"] = {f"out{i}": o.cpu() for i, o in enumerate(outs)}
                res[f"{name}.B{b}.T{t}"]["workspace_bytes"] = torch.tensor(asked)
    torch.save(res, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="root of the other checkout (built)")
    ap.add_argument("--_run", nargs=2, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args._run:
        run(*args._run)
        return
    import torch

    with tempfile.TemporaryDirectory() as tmp:
        outs = []
        for i, tree in enumerate((ROOT, os.path.abspath(args.other))):
            out = os.path.join(tmp, f"{i}.pt")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--other", args.other, "--_run", tree, out])
            outs.append(torch.load(out))
    eq = {f"{kind}.{k}": torch.equal(outs[0][kind][k], outs[1][kind][k]) for kind in outs[0] for k in outs[0][kind]
          if k != "workspace_bytes"}
    ws = {kind: list(zip(outs[0][kind]["workspace_bytes"].tolist(), outs[1][kind]["workspace_bytes"].tolist()))
          for kind in outs[0]}
    print(json.dumps({"equal": all(eq.values()), "outputs": eq, "workspace_bytes": ws}))


if __name__ == "__main__":
    main()
