"""Recorded reference results for the tests that compare with the unmodified reference project.

A test names what the reference computes (a state-dict layout, a value, an output tensor) with a function that computes
it from the reference.  Where the reference tree is importable that function runs and the test compares live; with
TTS_WRITE_GOLDEN=1 set as well, the result is stored under tests/golden/reference/<test>.pt (tests/golden/make_golden.py
does this for every such test).  Where the reference is absent the stored result stands in for it, so the comparison
runs on every machine.  Large tensors are stored as a fixed, seeded sample of their elements (0/1 tensors exactly, as
packed bits) to keep each file small.

Weights are never stored: `seeded_state_dict` draws every floating-point entry of a state-dict layout from a seeded
generator, and the live path loads the same values into the reference module."""
import math
import os

import numpy as np
import torch

import ref_import

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIR = os.path.join(ROOT, "tests", "golden", "reference")
SAMPLE = 8192          # elements kept of a tensor larger than this


def live() -> bool:
    return ref_import.available()


def layout(state_dict):
    """[(key, shape, dtype, value)] of a state dict; value only for non-floating-point entries."""
    return [(k, tuple(v.shape), str(v.dtype), None if v.is_floating_point() else v.clone()) for k, v in state_dict.items()]


def seeded_state_dict(spec, seed):
    """Deterministic weights for a state-dict layout: uniform(+-1/sqrt(fan_in)) for tensors of rank >= 2 (PyTorch's
    default conv / linear scale), 1 + N(0, 0.05) for normalisation gains, N(0, 0.05) for every other vector."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, shape, dtype, value in spec:
        if value is not None:
            out[k] = value.clone()
            continue
        if len(shape) >= 2:
            b = 1.0 / math.sqrt(max(1, math.prod(shape[1:])))
            t = (torch.rand(shape, generator=g) * 2 - 1) * b
        else:
            t = torch.randn(shape, generator=g) * 0.05
            if k.endswith("gamma") or k.endswith("norm.weight") or (".norms" in k and k.endswith("weight")):
                t = t + 1.0
        out[k] = t.to(getattr(torch, dtype.replace("torch.", "")))
    return out


def _pack(t):
    t = t.detach().cpu()
    if t.numel() <= SAMPLE:
        return {"full": t.clone()}
    flat = t.reshape(-1)
    if t.is_floating_point() and bool(((flat == 0) | (flat == 1)).all()):
        return {"shape": tuple(t.shape), "dtype": str(t.dtype), "bits": torch.from_numpy(np.packbits(flat.numpy() == 1))}
    idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:SAMPLE]
    return {"shape": tuple(t.shape), "dtype": str(t.dtype), "sample": flat[idx].clone()}


def _matches(got, rec, atol):
    got = got.detach().cpu()
    if "full" in rec:
        want = rec["full"]
        if got.shape != want.shape:
            return False
        return torch.equal(got, want) if atol is None else torch.allclose(got, want, atol=atol, rtol=0)
    if tuple(got.shape) != tuple(rec["shape"]) or str(got.dtype) != rec["dtype"]:
        return False
    flat = got.reshape(-1)
    if "bits" in rec:
        want = torch.from_numpy(np.unpackbits(rec["bits"].numpy())[: flat.numel()].astype(np.float32)).to(flat.dtype)
    else:
        idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:SAMPLE]
        flat, want = flat[idx], rec["sample"]
    return torch.equal(flat, want) if atol is None else torch.allclose(flat, want, atol=atol, rtol=0)


class Recorded:
    """Reference results of one test: live where the reference exists, from tests/golden/reference/<name>.pt otherwise."""

    def __init__(self, name):
        self.path = os.path.join(DIR, name + ".pt")
        self.live = live()
        self.write = self.live and os.environ.get("TTS_WRITE_GOLDEN") == "1"
        self.data = {}
        if not self.live:
            assert os.path.exists(self.path), f"no reference tree and no recorded results in {self.path}"
            self.data = torch.load(self.path, map_location="cpu", weights_only=False)

    def value(self, key, fn):
        """A small reference-side value (layout, ids, config fields, shapes): fn() live, the stored value otherwise."""
        if not self.live:
            return self.data[key]
        v = fn()
        self.data[key] = v
        return v

    def check(self, key, got, fn, atol=None):
        """Asserts that `got` equals the reference's tensor fn() (allclose with `atol` when given)."""
        if self.live:
            want = fn()
            ok = torch.equal(got, want) if atol is None else torch.allclose(got, want, atol=atol, rtol=0)
            assert ok, key
            self.data[key] = _pack(want)
        else:
            assert _matches(got, self.data[key], atol), key

    def save(self):
        if self.write:
            os.makedirs(DIR, exist_ok=True)
            torch.save(self.data, self.path)
