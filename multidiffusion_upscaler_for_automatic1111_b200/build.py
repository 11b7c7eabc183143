"""Build recipe for libtd_b200.so (hand-written sm_90a CUDA behind a C-ABI).

`nvcc` cross-compiles without a GPU, so the library can be built on a machine without one; it is
git-ignored and written next to this file.  Usage: `python -m multidiffusion_upscaler_for_automatic1111_b200.build`.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
INCLUDE = os.path.join(os.path.dirname(PKG_DIR), "include")
LIB_PATH = os.path.join(PKG_DIR, "libtd_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def _deps():
    out = sources()
    out += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    out += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE) if f.endswith(".h")]
    out.append(os.path.abspath(__file__))
    return out


def needs_build() -> bool:
    if not os.path.isfile(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(p) > t for p in _deps())


def build_variant(out_path: str, defines) -> str:
    """Tuning aid: the same sources with extra -D knobs (TD_AS_ROWS, TD_AS_X, TD_AS_PPC ...) into `out_path`;
    load it with TD_B200_LIB=<out_path> (bench.py, tests).  Never replaces the default library."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    os.makedirs(os.path.dirname(os.path.abspath(out_path)) or ".", exist_ok=True)
    flags = [f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")]
    cmd = [nvcc, *flags, *[f"-D{d}" for d in defines], "-I", INCLUDE, "-I", CSRC, "-o", out_path, *sources()]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + (res.stdout + res.stderr)[-8000:])
    return out_path


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into libtd_b200.so; returns its path."""
    if not force and not needs_build():
        return LIB_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libtd_b200.so (no CPU fallback exists)")
    tmp = LIB_PATH + ".tmp"
    cmd = [nvcc, *NVCC_FLAGS, "-I", INCLUDE, "-I", CSRC, "-o", tmp, *sources()]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(PKG_DIR, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + log[-8000:])
    os.replace(tmp, LIB_PATH)
    if verbose:
        print(log)
    return LIB_PATH


if __name__ == "__main__":
    if "--variant" in sys.argv:      # python build.py --variant build/variants/libtd_x16.so TD_AS_X=16 TD_AS_PPC=1
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], sys.argv[i + 2:]))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
