"""Builds ``lib/libsrcv_b200.so`` in-tree with nvcc for sm_90a.

    python -m simplerecon_b200.build [--force] [--verbose]

Plain ``nvcc -shared`` (no torch headers: the library is a C ABI, torch only
supplies device memory and streams at run time).  The .so is a build product
(git-ignored); ``__graft_entry__.build()`` recreates it when a source is newer.
"""
from __future__ import annotations

import argparse
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
SRC = sorted((PKG / "csrc").glob("*.cu"))
HDR = sorted((PKG / "csrc").glob("*.cuh")) + sorted((PKG / "csrc").glob("*.h")) + \
    [PKG.parent / "include" / "srcv_b200.h"]
OUT = PKG / "lib" / "libsrcv_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]
# Preprocessor switches of the shipped build.  tests/emu compiles the same sources with the same
# list, so the host emulation (parity, TSan, fuzzing) validates the binary that ships.
NVCC_DEFINES: list[str] = []


def nvcc_path() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and Path(c).is_file():
            return c
    raise RuntimeError("nvcc not found")


def up_to_date() -> bool:
    if not OUT.is_file():
        return False
    t = OUT.stat().st_mtime
    return all(p.stat().st_mtime <= t for p in SRC + HDR)


def build(force: bool = False, verbose: bool = False, out: Path | None = None, extra: list[str] | None = None) -> Path:
    """``out`` / ``extra`` build an experiment variant next to the default library (e.g.
    ``--out lib/libsrcv_b200_uw.so --extra=-DSRCV_TC_UNIFORM_WARP``; load it with
    ``SRCV_B200_LIB=<path>``); the default build never takes extra flags."""
    if out is None and not extra and not force and up_to_date():
        return OUT
    out = Path(out) if out else OUT
    out.parent.mkdir(parents=True, exist_ok=True)
    cmd = [nvcc_path(), *NVCC_FLAGS, *NVCC_DEFINES, *(extra or []), *(["-Xptxas", "-v"] if verbose else []),
           "-o", str(out), *map(str, SRC)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed ({r.returncode}): {' '.join(cmd)}")
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--out", default=None, help="write an experiment variant here instead of the default library")
    ap.add_argument("--extra", action="append", default=[], help="extra nvcc flag (repeatable), variants only")
    a = ap.parse_args()
    print(build(a.force, a.verbose, a.out, a.extra))
