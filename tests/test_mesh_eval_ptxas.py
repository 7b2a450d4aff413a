"""CPU tier: what ptxas makes of the mesh-evaluation kernels (csrc/srcv_mesh_eval.cuh, DESIGN §4.17), and that moving
the cell hash into srcv_block_hash.cuh left the voxel-block TSDF kernels' machine code as it was.

Compiles ``srcv_tsdf.cu`` (which includes the sparse TSDF and mesh-evaluation headers) with the shipped flags and
``-Xptxas -v``: every mesh-evaluation kernel has no spills and no stack.  The sparse TSDF kernels' SASS must not
depend on where the hash helpers are defined: the unit compiled with the helpers inlined back into
srcv_tsdf_sparse.cuh (their definitions before the move, restated below) gives byte-identical SASS for every sparse
kernel.  Needs nvcc, not a GPU.
"""
from __future__ import annotations

import re
import shutil
import subprocess
from pathlib import Path

import pytest

from simplerecon_b200 import build as B

CSRC = B.PKG / "csrc"


def _nvcc():
    try:
        return B.nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")


def _compile(src_dir, out, extra=()):
    flags = [f for f in B.NVCC_FLAGS if f != "-shared"]
    cmd = [_nvcc(), *flags, *B.NVCC_DEFINES, *extra, "-cubin", "-o", str(out), str(src_dir / "srcv_tsdf.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed:\n{r.stderr[-4000:]}"
    return r.stdout + r.stderr


@pytest.fixture(scope="module")
def ptxas_props(tmp_path_factory) -> dict:
    log = _compile(CSRC, tmp_path_factory.mktemp("ptxas") / "srcv_tsdf.cubin", ["-Xptxas", "-v"])
    return {name: (int(stack), int(st), int(ld)) for name, stack, st, ld in re.findall(
        r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
        log)}


MESH_EVAL_KERNELS = ("area_kernel", "scan_tiles_kernel", "scan_offsets_kernel", "scan_apply_kernel", "sample_kernel",
                     "bbox_kernel", "grid_params_kernel", "grid_clear_kernel", "grid_count_kernel",
                     "grid_scatter_kernel", "near_kernel", "brute_kernel", "dist_out_kernel", "reduce_kernel",
                     "metrics_finalize_kernel")


@pytest.mark.parametrize("kernel", MESH_EVAL_KERNELS)
def test_mesh_eval_kernels_no_spills_no_stack(ptxas_props, kernel):
    hits = {k: v for k, v in ptxas_props.items() if "mesh_eval_detail" in k and kernel in k}
    assert hits, f"no {kernel} in the ptxas output"
    for name, props in hits.items():
        assert props == (0, 0, 0), f"{name}: stack {props[0]}, spill stores {props[1]}, spill loads {props[2]}"


# the hash helpers as srcv_tsdf_sparse.cuh defined them before they moved to srcv_block_hash.cuh
_INLINE_HASH = '''namespace srcv {
namespace {
#ifdef SRCV_HOST_EMU
inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED);
  return cmp;
}
inline unsigned long long load_key(const unsigned long long* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
#else
__device__ __forceinline__ unsigned long long load_key(const unsigned long long* p) {
  return *reinterpret_cast<const volatile unsigned long long*>(p);
}
#endif
constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int kKeyBias = 1 << 20;
__device__ __forceinline__ bool block_in_range(int bx, int by, int bz) {
  return bx >= -kKeyBias && bx < kKeyBias && by >= -kKeyBias && by < kKeyBias && bz >= -kKeyBias && bz < kKeyBias;
}
__device__ __forceinline__ unsigned long long block_key(int bx, int by, int bz) {
  return ((unsigned long long)(unsigned)(bx + kKeyBias) << 42) | ((unsigned long long)(unsigned)(by + kKeyBias) << 21) |
         (unsigned long long)(unsigned)(bz + kKeyBias);
}
__device__ __forceinline__ unsigned block_hash(unsigned long long k, unsigned mask) {
  k ^= k >> 31; k *= 0x7fb5d329728ea185ull;
  k ^= k >> 27; k *= 0x81dadef4bc2dd44dull;
  k ^= k >> 33;
  return (unsigned)k & mask;
}
}  // namespace
}  // namespace srcv
'''


def _sparse_sass(cubin) -> dict:
    cuobjdump = shutil.which("cuobjdump") or str(Path(_nvcc()).parent / "cuobjdump")
    r = subprocess.run([cuobjdump, "-sass", str(cubin)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    parts = re.split(r"\n\s*Function : (\S+)\n", r.stdout)
    return {parts[i]: re.sub(r"/\*[0-9a-f]{4,}\*/", "", parts[i + 1]) for i in range(1, len(parts), 2)
            if "sparse" in parts[i] or "SparseMeshParams" in parts[i]}


def test_sparse_tsdf_sass_unchanged_by_the_hash_move(tmp_path):
    """The unit as shipped against a copy in which srcv_tsdf_sparse.cuh defines the helpers itself and the
    mesh-evaluation header is left out: the same sparse kernels, instruction for instruction."""
    old = tmp_path / "pkg" / "csrc"                  # srcv_kernels.h includes ../../include/srcv_b200.h
    shutil.copytree(CSRC, old)
    sparse = (old / "srcv_tsdf_sparse.cuh").read_text()
    assert '#include "srcv_block_hash.cuh"\n' in sparse
    sparse = sparse.replace('#include "srcv_block_hash.cuh"\n', "")
    head, sep, tail = sparse.partition("namespace srcv {\n")
    (old / "srcv_tsdf_sparse.cuh").write_text(head + _INLINE_HASH + sep + tail)
    tsdf = (old / "srcv_tsdf.cu").read_text()
    (old / "srcv_tsdf.cu").write_text(tsdf.replace('#include "srcv_mesh_eval.cuh"', ""))
    (old / "srcv_block_hash.cuh").unlink()
    (tmp_path / "include").mkdir()
    shutil.copy(B.PKG.parent / "include" / "srcv_b200.h", tmp_path / "include")
    _compile(CSRC, tmp_path / "new.cubin")
    _compile(old, tmp_path / "old.cubin")
    new, ref = _sparse_sass(tmp_path / "new.cubin"), _sparse_sass(tmp_path / "old.cubin")
    assert len(ref) >= 12, sorted(ref)
    # the anonymous namespace's mangled name depends on the file path: compare by kernel, not by symbol
    strip = lambda d: {re.sub(r"_GLOBAL__N__[0-9a-f_]+_srcv_tsdf_cu_[0-9a-f]+", "", k): v for k, v in d.items()}
    new, ref = strip(new), strip(ref)
    assert sorted(new) == sorted(ref)
    for k in ref:
        assert new[k] == ref[k], f"{k}: SASS differs after the hash move"
