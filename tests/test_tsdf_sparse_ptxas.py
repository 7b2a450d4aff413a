"""CPU tier: what ptxas makes of the voxel-block TSDF kernels (DESIGN §4.16).

Compiles ``srcv_tsdf.cu`` (which includes ``srcv_tsdf_sparse.cuh``) with the shipped flags and ``-Xptxas -v``.
The allocation, update, read-back and table kernels have no spills and no stack.  The mesh kernels instantiated on
the voxel-block view keep the IEEE division's slow-path call of the dense mesh kernels; registers live across that
call may cost a few bytes of stack, bounded here so that a change that spills the hot loop shows up.  The dense
kernels of the unit keep no spills where they had none.  Needs nvcc, not a GPU.
"""
from __future__ import annotations

import re
import subprocess

import pytest

from simplerecon_b200 import build as B


@pytest.fixture(scope="module")
def ptxas_props(tmp_path_factory) -> dict:
    try:
        nvcc = B.nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "srcv_tsdf.o"
    flags = [f for f in B.NVCC_FLAGS if f != "-shared"]
    cmd = [nvcc, *flags, *B.NVCC_DEFINES, "-c", "-Xptxas", "-v", "-o", str(out), str(B.PKG / "csrc" / "srcv_tsdf.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed:\n{r.stderr[-4000:]}"
    log = r.stdout + r.stderr
    return {name: (int(stack), int(st), int(ld)) for name, stack, st, ld in re.findall(
        r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
        log)}


SPARSE_KERNELS = ("sparse_reset_kernel", "sparse_tile_depth_kernel", "sparse_alloc_kernel", "sparse_integrate_kernel",
                  "sparse_read_box_kernel", "sparse_boundary_kernel", "sparse_release_kernel", "sparse_neighbour_kernel")


@pytest.mark.parametrize("kernel", SPARSE_KERNELS)
def test_sparse_kernels_no_spills_no_stack(ptxas_props, kernel):
    hits = {k: v for k, v in ptxas_props.items() if kernel in k}
    assert hits, f"no {kernel} in the ptxas output"
    for name, props in hits.items():
        assert props == (0, 0, 0), f"{name}: stack {props[0]}, spill stores {props[1]}, spill loads {props[2]}"


def test_sparse_mesh_kernels_stack_bounded(ptxas_props):
    hits = {k: v for k, v in ptxas_props.items() if "SparseMeshParams" in k}
    assert len(hits) == 4, sorted(hits)
    for name, (stack, st, ld) in hits.items():
        assert stack <= 64 and st <= 64 and ld <= 64, f"{name}: stack {stack}, spill stores {st}, spill loads {ld}"


def test_dense_integration_kernels_no_spills(ptxas_props):
    hits = {k: v for k, v in ptxas_props.items() if "tsdf_integrate" in k}
    assert len(hits) == 4
    for name, props in hits.items():
        assert props == (0, 0, 0), f"{name}: {props}"
