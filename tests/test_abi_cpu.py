"""CPU-only checks of the C-ABI libraries: they build, load, and export every symbol the
headers declare; without a CUDA device the engine refuses loudly (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

from rucene_b200 import _build, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header, prefix):
    txt = open(os.path.join(ROOT, "include", header)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(%s[a-z0-9_]+)\s*\(" % prefix, txt)))


def test_gpu_library_exports_every_declared_symbol():
    L = C.CDLL(_build.build_gpu())
    names = _declared("rucene_gpu.h", "rg_")
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), n


def test_codec_library_exports_every_declared_symbol():
    L = C.CDLL(_build.build_codec())
    names = _declared("rucene_codec.h", "rc_")
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), n


def test_engine_fails_loudly_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(engine.EngineError) as ei:
        engine.Engine()
    assert ei.value.code == engine.RG_ENODEVICE
    assert "no CPU fallback" in str(ei.value)


def test_gpu_library_targets_sm_90a():
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-lelf", _build.build_gpu()], stdout=subprocess.PIPE, text=True).stdout
    assert "sm_90a" in out
