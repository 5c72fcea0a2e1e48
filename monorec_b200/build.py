"""Builds libmonorec_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache: the .so sits next to the package).

    python -m monorec_b200.build [--force] [--verbose]
"""
import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libmonorec_b200.so"
STAMP = PKG / ".libmonorec_b200.stamp"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17"]


def sources():
    return sorted(CSRC.glob("*.cu"))


def _digest():
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "monorec_b200.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    dig = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == dig:
        return LIB
    if not Path(NVCC).exists():
        if LIB.exists() and os.environ.get("MONOREC_B200_ALLOW_STALE") == "1":
            import warnings
            warnings.warn(f"{LIB.name} does not match the sources (digest mismatch) and nvcc is missing: using the stale "
                          "library because MONOREC_B200_ALLOW_STALE=1")
            return LIB
        raise RuntimeError(f"nvcc not found at {NVCC} and {LIB.name} is missing or older than the sources "
                           "(set MONOREC_B200_ALLOW_STALE=1 to load a stale library anyway)")
    cmd = [NVCC, *FLAGS, "-shared", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2"]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += ["-o", str(LIB)] + [str(s) for s in sources()]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libmonorec_b200.so")
    STAMP.write_text(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
