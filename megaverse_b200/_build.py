"""In-tree build of the native code (no JIT cache: the built .so files travel to the GPU box with the repo snapshot).

  libmegaverse_b200.so                         C-ABI engine: sm_90a (H100) kernels + host level generation   (nvcc)
  extension/megaverse.cpython-*.so             pybind11 module `megaverse_b200.extension.megaverse`           (g++)
"""
import os
import shutil
import subprocess
import sys
import sysconfig

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libmegaverse_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    # no FMA contraction on either side: device results must equal a plain IEEE CPU evaluation (parity with the oracle)
    "-fmad=false", "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(ROOT, "include", "megaverse_b200.h")]


def ext_path():
    suffix = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return os.path.join(PKG, "extension", "megaverse" + suffix)


def build_lib(force=False, verbose=False):
    srcs = _sources()
    if not force and _newer(LIB, srcs):
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    extra = os.environ.get("MV_NVCC_EXTRA", "").split()  # developer switches, e.g. -DMV_KCC_COUNTERS
    # state_copy.cu and ray_kernel.cu are modules of their own: NVVM optimises per module, so the engine's kernels do not see them
    srcs = ("engine.cu", "state_copy.cu", "ray_kernel.cu", "levelgen.cpp")
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + [os.path.join(CSRC, f) for f in srcs]
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB


def build_ext(force=False):
    import pybind11

    out = ext_path()
    src = os.path.join(CSRC, "pybind_module.cpp")
    if not os.path.exists(src):
        return None
    if not force and _newer(out, [src, LIB, os.path.join(ROOT, "include", "megaverse_b200.h")]):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cmd = [
        os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden",
        "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"], "-I", os.path.join(ROOT, "include"),
        src, "-o", out, "-L", PKG, "-lmegaverse_b200", "-Wl,-rpath,$ORIGIN/..",
    ]
    subprocess.check_call(cmd)
    return out


def build_all(force=False, verbose=False):
    build_lib(force, verbose)
    build_ext(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built", LIB, ext_path())
