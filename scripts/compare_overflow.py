#!/usr/bin/env python
"""Overflow / Neural-HMM outputs of this tree against another build of the package, on the same seeded inputs.

    python scripts/compare_overflow.py --other /path/to/other/checkout   (both trees built with __graft_entry__.build())

Runs the same three workloads in each tree, each in a subprocess with that tree first on sys.path: Overflow at
temperature 0, Neural-HMM without prenet dropout, and Overflow sampled at 0.334 with supplied noise, 12 ragged rows of
20-59 tokens with the seeded test weights (tests/overflow_oracle.py).  Prints one JSON line with ``torch.equal`` per
output and ``"equal": true`` when every output matches bit for bit.  Used to show that moving Overflow's kernels into
the shared recurrent unit left its results unchanged.  Writes only to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(tree, out):
    import torch

    sys.path[:0] = [tree, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]
    import overflow_oracle as OO
    from ref_golden import layout, seeded_state_dict
    from tts_b200 import overflow as OV

    assert os.path.realpath(OV.__file__).startswith(os.path.realpath(tree)), OV.__file__
    dev = torch.device("cuda:0")
    res = {}
    for kind, over in (("overflow", dict(sampling_temp=0.0)), ("neuralhmm", dict(prenet_dropout_at_inference=False)),
                       ("overflow_sampled", dict(sampling_temp=0.334))):
        cls, ccls = (OV.Overflow, OV.OverflowConfig) if kind.startswith("overflow") else \
            (OV.NeuralhmmTTS, OV.NeuralhmmTTSConfig)
        cfg = ccls(num_chars=40, **over)
        m = cls(cfg)
        sd = OO.seeded_weights(seeded_state_dict(layout(m.state_dict()), 13), 17)
        m.load_state_dict(sd)
        m.eval().to(dev)
        g = torch.Generator().manual_seed(3)
        lens = torch.randint(20, 60, (12,), generator=g)
        text = torch.zeros(12, int(lens.max()), dtype=torch.long)
        for b, n in enumerate(lens.tolist()):
            text[b, :n] = torch.randint(1, 40, (n,), generator=g)
        draws = {"noise": torch.randn(12, cfg.max_sampling_time, 80, generator=g).to(dev)}
        o = m.inference(text.to(dev), {"x_lengths": lens.to(dev)}, draws=draws)
        res[kind] = {k: v.cpu() for k, v in o.items() if torch.is_tensor(v)}
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
    eq = {f"{kind}.{k}": torch.equal(outs[0][kind][k], outs[1][kind][k]) for kind in outs[0] for k in outs[0][kind]}
    print(json.dumps({"equal": all(eq.values()), "outputs": eq}))


if __name__ == "__main__":
    main()
