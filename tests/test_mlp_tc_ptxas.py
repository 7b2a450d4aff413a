"""CPU tier: what ptxas makes of the wgmma sweep kernel.

Compiles ``srcv_mlp_tc.cu`` with the shipped flags (``build.NVCC_FLAGS`` + ``NVCC_DEFINES``) and
``-Xptxas -v`` and checks every ``mlp_tc_kernel`` instantiation: no C7512 (ptxas serialising the
wgmma chains for lack of registers, so that every MMA waits for the previous one) and no register
spills.  Either would quietly cost a large share of the sweep's time without changing a result,
so no numerical test notices it.  Needs nvcc, not a GPU.
"""
from __future__ import annotations

import re
import subprocess

import pytest

from simplerecon_b200 import build as B


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory) -> str:
    try:
        nvcc = B.nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "srcv_mlp_tc.o"
    flags = [f for f in B.NVCC_FLAGS if f != "-shared"]
    cmd = [nvcc, *flags, *B.NVCC_DEFINES, "-c", "-Xptxas", "-v", "-o", str(out),
           str(B.PKG / "csrc" / "srcv_mlp_tc.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed:\n{r.stderr[-4000:]}"
    return r.stdout + r.stderr


def _kernels(log: str) -> list[str]:
    names = re.findall(r"Compiling entry function '(\S*mlp_tc_kernel\S*)'", log)
    assert names, "no mlp_tc_kernel instantiation in the ptxas output"
    return names


def test_wgmma_chains_not_serialised(ptxas_log):
    serialised = set(re.findall(r"\(C7512\)[^\n]*function '([^']+)'", ptxas_log))
    bad = [k for k in _kernels(ptxas_log) if k in serialised]
    assert not bad, f"ptxas serialises the wgmma chains (C7512) of {bad}"


def test_no_register_spills(ptxas_log):
    spills = {name: (int(st), int(ld)) for name, st, ld in re.findall(
        r"Function properties for (\S+)\n[^\n]*?(\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)}
    for k in _kernels(ptxas_log):
        assert k in spills, f"no spill line for {k}"
        assert spills[k] == (0, 0), f"{k}: {spills[k][0]} bytes spill stores, {spills[k][1]} bytes spill loads"
