"""tts_b200/csrc/build.sh fails, and links nothing, when a source file does not compile.

nvcc leaves the previous object on disk when a compile fails, so a build that only looked at the link step would link a
file's last good object and report success.  The test builds a throwaway tree twice: once with two good sources, then
after breaking one of them."""
import os
import shutil
import subprocess
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

GOOD = '#include "tiny.cuh"\nextern "C" int tiny_{name}() {{ return TINY + {n}; }}\n'


@pytest.fixture
def tree(tmp_path):
    if not os.path.exists(NVCC):
        pytest.skip(f"no nvcc at {NVCC}")
    csrc = tmp_path / "tts_b200" / "csrc"
    csrc.mkdir(parents=True)
    (tmp_path / "include").mkdir()
    shutil.copy(os.path.join(ROOT, "tts_b200", "csrc", "build.sh"), csrc / "build.sh")
    (tmp_path / "include" / "tts_b200.h").write_text("#pragma once\n")
    (csrc / "tiny.cuh").write_text("#pragma once\n#define TINY 1\n")
    (csrc / "a.cu").write_text(GOOD.format(name="a", n=1))
    (csrc / "b.cu").write_text(GOOD.format(name="b", n=2))
    return tmp_path


def build(tree):
    env = dict(os.environ, NVCC=NVCC)
    env.pop("PTXAS_V", None)
    return subprocess.run(["bash", str(tree / "tts_b200" / "csrc" / "build.sh")], env=env, capture_output=True,
                          text=True, timeout=600)


def test_a_failed_compile_fails_the_build_and_links_nothing(tree):
    so = tree / "tts_b200" / "libtts_b200.so"
    stale = tree / "build" / "obj" / "b.o"
    first = build(tree)
    assert first.returncode == 0, first.stderr
    assert so.exists() and stale.exists()
    so.unlink()
    bad = tree / "tts_b200" / "csrc" / "b.cu"
    bad.write_text('extern "C" int tiny_b( { return 2; }\n')   # a syntax error
    later = time.time() + 10                                   # newer than b.o whatever the clock's resolution
    os.utime(bad, (later, later))
    second = build(tree)
    assert second.returncode != 0, second.stdout
    assert not so.exists(), "linked a library from a failed build"
    assert not stale.exists(), "kept the object of the file that failed to compile"
