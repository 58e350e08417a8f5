"""The C-ABI library builds, loads, and exports every symbol include/tts_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "tts_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200tts_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_something():
    syms = declared_symbols()
    assert "b200tts_mas" in syms and "b200tts_hifigan_forward" in syms


def test_library_exports_every_declared_symbol():
    path = os.path.join(ROOT, "tts_b200", "libtts_b200.so")
    assert os.path.exists(path), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(path)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"declared in include/tts_b200.h but not exported: {missing}"
    lib.b200tts_version.restype = ctypes.c_int
    assert lib.b200tts_version() >= 100


def test_library_exports_the_device_buffer_counter():
    from tts_b200 import _lib

    lib = _lib.lib()
    assert hasattr(lib, "b200tts_debug_device_buffers")
    assert lib.b200tts_debug_device_buffers.restype is ctypes.c_longlong
    assert lib.b200tts_debug_device_buffers() >= 0


def test_product_fails_loudly_without_cuda():
    import pytest
    import torch

    from tts_b200.helpers import maximum_path

    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    with pytest.raises(RuntimeError, match="no CPU path"):
        maximum_path(torch.zeros(1, 2, 3), torch.ones(1, 2, 3))
