"""CPU tier: what ptxas makes of the voxel down-sampling kernels (csrc/srcv_voxel_downsample.cuh, DESIGN §4.19).

Compiles ``srcv_tsdf.cu`` (which includes the mesh-evaluation headers and this one) with the shipped flags and
``-Xptxas -v``: every voxel down-sampling kernel has no spills and no stack.  Needs nvcc, not a GPU.
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
    flags = [f for f in B.NVCC_FLAGS if f != "-shared"]
    out = tmp_path_factory.mktemp("ptxas") / "srcv_tsdf.cubin"
    r = subprocess.run([nvcc, *flags, *B.NVCC_DEFINES, "-Xptxas", "-v", "-cubin", "-o", str(out),
                        str(B.PKG / "csrc" / "srcv_tsdf.cu")], capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed:\n{r.stderr[-4000:]}"
    return {name: (int(stack), int(st), int(ld)) for name, stack, st, ld in re.findall(
        r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
        r.stdout + r.stderr)}


VOXEL_KERNELS = ("params_kernel", "key_kernel", "radix_hist_kernel", "radix_scatter_kernel", "head_kernel",
                 "start_kernel", "mean_kernel")


@pytest.mark.parametrize("kernel", VOXEL_KERNELS)
def test_voxel_kernels_no_spills_no_stack(ptxas_props, kernel):
    hits = {k: v for k, v in ptxas_props.items() if "voxel_ds_detail" in k and kernel in k}
    assert hits, f"no {kernel} in the ptxas output"
    for name, props in hits.items():
        assert props == (0, 0, 0), f"{name}: stack {props[0]}, spill stores {props[1]}, spill loads {props[2]}"


def test_unsigned_scan_of_the_sort_no_spills(ptxas_props):
    hits = {k: v for k, v in ptxas_props.items() if "mesh_eval_detail" in k and "scan_" in k and "IjE" in k}
    assert len(hits) == 3, sorted(hits)
    assert all(v == (0, 0, 0) for v in hits.values())
