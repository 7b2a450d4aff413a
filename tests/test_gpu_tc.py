"""GPU: the wgmma building block on its own — D = A W^T with A (fp16 hi/lo split) and the
core-matrix weights in shared memory, three MMAs per K step — against an fp64 matmul.  Pins the
core-matrix packing order, the shared-memory descriptors and the accumulator fragment layout the
metadata-MLP kernel uses."""
import ctypes as C

import pytest
import torch

from simplerecon_b200 import _native

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("Kp,scale", [(16, 1.0), (64, 1.0), (128, 1.0), (208, 1.0), (208, 30.0), (256, 1e-3)])
def test_tc_gemm_matches_fp64(cuda_device, built_lib, Kp, scale):
    g = torch.Generator().manual_seed(Kp)
    A = (torch.randn(128, Kp, generator=g) * scale).to(cuda_device)
    Wm = (torch.rand(128, Kp, generator=g) * 2 - 1).mul(0.07).to(cuda_device)
    D = torch.full((128, 128), float("nan"), device=cuda_device)
    scratch = torch.empty(512 * Kp, dtype=torch.uint8, device=cuda_device)
    st = built_lib.srcv_tc_selftest_f32(A.data_ptr(), Wm.data_ptr(), Kp, D.data_ptr(), scratch.data_ptr(),
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream))
    _native.check(st)
    torch.cuda.synchronize()
    ref = A.double() @ Wm.double().t()
    err = (D.double() - ref).abs().max().item()
    # fp32 product noise: |A||W| sqrt(K) 2^-22-ish; fp32 matmul itself is no better
    ref32 = (A @ Wm.t()).double()
    e32 = (ref32 - ref).abs().max().item()
    # ... plus the fp16-subnormal floor of the lo halves (|x| < ~0.1 keeps an absolute 3e-8)
    bound = 4 * max(e32, 1e-7 * float(ref.abs().max())) + 6e-8 * 0.07 * Kp ** 0.5 * 2
    assert err <= bound, f"wgmma GEMM err {err:.3e} (fp32 matmul err {e32:.3e})"


def test_tc_gemm_structured_operands(cuda_device, built_lib):
    """Identity-like operands expose any permutation of rows / K positions exactly."""
    Kp = 128
    A = torch.zeros(128, Kp)
    Wm = torch.zeros(128, Kp)
    for r in range(128):
        A[r, r % Kp] = r + 1                 # row r has one non-zero at K = r
        Wm[r, (r * 7) % Kp] = 0.5 + r        # weight row n has one non-zero at K = 7n mod 128
    A, Wm = A.to(cuda_device), Wm.to(cuda_device)
    D = torch.empty(128, 128, device=cuda_device)
    scratch = torch.empty(512 * Kp, dtype=torch.uint8, device=cuda_device)
    _native.check(built_lib.srcv_tc_selftest_f32(A.data_ptr(), Wm.data_ptr(), Kp, D.data_ptr(),
                                                 scratch.data_ptr(), None))
    torch.cuda.synchronize()
    assert torch.equal(D, A @ Wm.t())        # small integers / halves: exact in every format
