"""In-tree build of the native pieces (no JIT cache: the built .so files travel to the GPU box).

  host/{loader,synth,result_io}.cc       ->  karpenter-core_b200/libkmodel.so   (string-level model: JSON loader, synthetic BASELINE
                                             configurations, result accessors - no CUDA, no solver; the oracle's tests and the
                                             bench's reference arm load this one alone)
  csrc/ksched.cu + host/{encoder,scheduler}.cc  ->  karpenter-core_b200/libksched.so   (C-ABI of include/ksched.h + host layer)
"""
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

MODEL_SRCS = ["loader.cc", "synth.cc", "result_io.cc"]
HOST_SRCS = ["encoder.cc", "scheduler.cc"]
CUDA_SRCS = ["ksched.cu"]


def _newer(target: Path, sources) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in sources)


def _run(cmd):
    print("+", " ".join(str(c) for c in cmd), flush=True)
    subprocess.check_call([str(c) for c in cmd])


def build_product(force=False, verbose_ptxas=False):
    out = PKG / "libksched.so"
    srcs = [PKG / "host" / s for s in HOST_SRCS] + [PKG / "csrc" / s for s in CUDA_SRCS]
    deps = srcs + list((PKG / "host").glob("*.h")) + list((PKG / "csrc").glob("*.cuh")) + list((ROOT / "include").glob("*.h"))
    deps.append(Path(__file__))  # the flags (ARCH) live in this file
    if not force and not _newer(out, deps):
        return out
    cmd = [NVCC, *ARCH, "-O3", "-std=c++17", "-lineinfo", "-shared", "-Xcompiler", "-fPIC,-Wall",
           "-I", ROOT / "include", "-I", PKG / "host", "-I", PKG / "csrc", "-o", out, *srcs, "-lnccl"]
    if verbose_ptxas:
        cmd.insert(1, "-Xptxas=-v")
    if os.environ.get("KSCHED_PROFILE_K1"):
        cmd.insert(1, "-DKSCHED_PROFILE_K1")
    if os.environ.get("KSCHED_PROFILE_PACK"):
        cmd.insert(1, "-DKSCHED_PROFILE_PACK")
    _run(cmd)
    return out


def build_model(force=False):
    out = PKG / "libkmodel.so"
    srcs = [PKG / "host" / s for s in MODEL_SRCS]
    deps = srcs + list((PKG / "host").glob("*.h")) + [Path(__file__)]  # the flags (ARCH) live in this file
    if not force and not _newer(out, deps):
        return out
    # linked by nvcc's host toolchain like libksched.so (shared libstdc++): objects of one library are read by the other
    _run([NVCC, *ARCH, "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-Wall", "-I", PKG / "host", "-o", out, *srcs])
    return out


def build_all(force=False):
    build_model(force)
    build_product(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)
