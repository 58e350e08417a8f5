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


def test_library_exports_the_debug_conv_layer():
    """the per-option conv aid (b200tts_debug_conv1d_*) is declared, exported and bound with its argument struct"""
    from tts_b200 import _lib

    syms = declared_symbols()
    assert "b200tts_debug_conv1d_create" in syms and "b200tts_debug_conv1d_launch" in syms
    lib = _lib.lib()
    assert lib.b200tts_debug_conv1d_create.restype is ctypes.c_int
    assert len(lib.b200tts_debug_conv1d_create.argtypes) == 10
    assert lib.b200tts_debug_conv1d_launch.argtypes[1] is ctypes.POINTER(_lib.DebugConvIOC)
    # the struct mirrors include/tts_b200.h field for field (x64 alignment: 8-byte pointers and long longs)
    src = open(os.path.join(ROOT, "include", "tts_b200.h")).read()
    body = re.search(r"typedef struct \{([^{}]*)\} b200tts_debug_conv_io;", src).group(1)
    names = re.findall(r"\*?\s*(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in _lib.DebugConvIOC._fields_]
    assert ctypes.sizeof(_lib.DebugConvIOC) == 216    # static_assert in capi.cu


def test_library_exports_the_debug_attention_and_layernorm():
    """the per-kernel transformer aids (b200tts_debug_attention / _add_layernorm) are declared, exported and bound"""
    from tts_b200 import _lib

    syms = declared_symbols()
    assert "b200tts_debug_attention" in syms and "b200tts_debug_add_layernorm" in syms
    lib = _lib.lib()
    vp, ci = ctypes.c_void_p, ctypes.c_int
    assert lib.b200tts_debug_attention.restype is ci
    assert lib.b200tts_debug_attention.argtypes == [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]
    assert lib.b200tts_debug_add_layernorm.restype is ci
    assert lib.b200tts_debug_add_layernorm.argtypes == [ci, vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ctypes.c_float, vp]
    # the bindings follow the header's parameter lists
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "tts_b200.h")).read(), flags=re.S)
    for name, n in (("b200tts_debug_attention", 11), ("b200tts_debug_add_layernorm", 13)):
        params = re.search(name + r"\(([^)]*)\);", src).group(1).split(",")
        assert len(params) == n == len(getattr(lib, name).argtypes), name
    assert "float eps" in re.search(r"b200tts_debug_add_layernorm\(([^)]*)\);", src).group(1).split(",")[11]


def test_product_fails_loudly_without_cuda():
    import pytest
    import torch

    from tts_b200.helpers import maximum_path

    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    with pytest.raises(RuntimeError, match="no CPU path"):
        maximum_path(torch.zeros(1, 2, 3), torch.ones(1, 2, 3))
