"""CPU tier: the host emulation's wgmma is asynchronous (tests/emu/emu_tc_async.h).

The emulated sweep kernel is only a check of its buffer hand-offs if an MMA reads its shared-memory
operands when a ``wgmma.wait_group`` retires it, not when it is issued.  One emulated warpgroup
checks exactly that: nothing is performed at issue or at commit, a store to the A operand between
issue and wait is what the MMA sees, and ``wait_group 1`` retires all groups but the newest.
"""
from __future__ import annotations

import shutil
import subprocess

import pytest

from tests import emu

PROGRAM = r"""
#include "emu_cuda.h"
#include "emu_tc_async.h"
#include <cstdio>
using namespace srcv::tc;

// A (64 x 16) at 0, B (128 x 16) at 2048: K-major no-swizzle core matrices, every element = v
static void fill(uint8_t* p, int rows, float v) {
  const uint16_t h = f16_sat_bits(v);
  for (int i = 0; i < rows * 16; ++i) std::memcpy(p + 2 * i, &h, 2);
}

int main() {
  std::atomic<int> errors{0};
  emu::launch(dim3(1), dim3(128), 2048 + 4096, [&] {
    uint8_t* sm = reinterpret_cast<uint8_t*>(emu::dynamic_smem());
    if (threadIdx.x == 0) { fill(sm, 64, 1.f); fill(sm + 2048, 128, 1.f); }
    __syncthreads();
    const uint64_t da = smem_desc(0, 64 * 16, 128), db = smem_desc(2048, 128 * 16, 128);
    float d[64], e[64];
    for (int i = 0; i < 64; ++i) d[i] = e[i] = -7.f;
    wgmma_ss_n128(d, da, db, 0u);
    wgmma_commit();
    if (d[0] != -7.f) errors++;                       // not performed at issue or commit
    __syncthreads();
    if (threadIdx.x == 0) fill(sm, 64, 2.f);          // the MMA has not read A yet
    __syncthreads();
    wgmma_ss_n128(e, da, db, 0u);
    wgmma_commit();
    wgmma_wait<1>();                                  // retires the first group only
    for (int i = 0; i < 64; ++i) if (d[i] != 32.f) errors++;   // 16 x (2 x 1): A read at the wait
    if (e[0] != -7.f) errors++;
    wgmma_wait<0>();
    for (int i = 0; i < 64; ++i) if (e[i] != 32.f) errors++;
  });
  std::printf("errors %d\n", errors.load());
  return errors.load() != 0;
}
"""


def test_wgmma_reads_shared_memory_at_the_wait(tmp_path):
    if not shutil.which(emu.CXX):
        pytest.skip("no host C++ compiler")
    src, exe = tmp_path / "async_wgmma.cpp", tmp_path / "async_wgmma"
    src.write_text(PROGRAM)
    r = subprocess.run([emu.CXX, "-std=c++20", "-pthread", "-O1", "-w", "-DSRCV_HOST_EMU=1", f"-I{emu.HERE}",
                        str(src), "-o", str(exe)], capture_output=True, text=True)
    if r.returncode != 0 and "c++20" in r.stderr:
        pytest.skip("host compiler without C++20")
    assert r.returncode == 0, r.stderr[-3000:]
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stdout + run.stderr
