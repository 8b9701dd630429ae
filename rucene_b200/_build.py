"""In-tree builds of the native libraries (no JIT cache: the .so files travel with the repo).

librucene_gpu.so   : CUDA kernels + the C ABI of include/rucene_gpu.h   (nvcc, sm_90a)
librucene_codec.so : host write side / BM25 host math / synthetic index (g++)

(The CPU checker under oracle/ is test infrastructure with its own Makefile; nothing in this
package builds, loads or mentions it.)
"""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rucene_b200")
LIB = os.path.join(PKG, "lib")
INC = os.path.join(ROOT, "include")

HOST_FLAGS = ["-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall",
              "-Wextra", "-pthread"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-ffp-contract=off,-pthread", "--fmad=false", "-prec-div=true",
              "-prec-sqrt=true", "-Xptxas", "-v"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _glob(d, exts):
    out = []
    for base, _dirs, files in os.walk(d):
        for f in files:
            if f.endswith(exts):
                out.append(os.path.join(base, f))
    return sorted(out)


def _run(cmd, log_name=None):
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log_name:
        os.makedirs(LIB, exist_ok=True)
        with open(os.path.join(LIB, log_name), "w") as f:
            f.write(" ".join(cmd) + "\n" + p.stdout)
    if p.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(cmd), p.stdout))
    return p.stdout


def codec_lib_path():
    return os.path.join(LIB, "librucene_codec.so")


def gpu_lib_path():
    return os.path.join(LIB, "librucene_gpu.so")


def build_codec(force=False):
    srcs = _glob(os.path.join(PKG, "csrc", "codec"), (".cpp",))
    deps = srcs + _glob(os.path.join(PKG, "csrc", "host"), (".hpp",)) + _glob(INC, (".h",))
    out = codec_lib_path()
    if force or _newer(out, deps):
        os.makedirs(LIB, exist_ok=True)
        cxx = shutil.which("g++") or "g++"
        _run([cxx] + HOST_FLAGS + ["-I" + INC, "-shared", "-o", out] + srcs, "build_codec.log")
    return out


def build_gpu(force=False):
    gdir = os.path.join(PKG, "csrc", "gpu")
    srcs = _glob(gdir, (".cu",))
    deps = srcs + _glob(gdir, (".cuh", ".h", ".hpp")) + _glob(os.path.join(PKG, "csrc", "host"), (".hpp",)) \
        + _glob(INC, (".h",))
    out = gpu_lib_path()
    if force or _newer(out, deps):
        os.makedirs(LIB, exist_ok=True)
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        _run([nvcc] + NVCC_FLAGS + ["-I" + INC, "-I" + gdir, "-shared", "-o", out] + srcs
             + ["-lcudart", "-ldl"], "build_gpu.log")
    return out


def build_all(force=False):
    return {"codec": build_codec(force), "gpu": build_gpu(force)}
