"""The product's SIMT kernels and C-ABI front end, compiled for the HOST (tests/emu: one
std::thread per CUDA thread, std::barrier for __syncthreads, NaN-poisoned shared memory)
and checked against the oracle — kernel-source parity in the CPU tier.

What this covers that the `-m gpu` tests cannot cover here (no GPU in this container):
indexing, barrier placement, launch heuristics (plane-loop split + last-arriver argmax of the
dot sweep, persistent grid of the MLP backward), workspace carving and argument validation of
every entry point of include/srcv_b200.h — including the wgmma kernel, which runs against a
functional model of wgmma / mbarrier / bulk copy (tests/emu/emu_tc.h).  What it
cannot cover: hardware limits, registers, speed, the asynchrony of wgmma — and device
intrinsics are replaced by IEEE host math, so tolerances are the parity tolerances of
tests/parity.py, not bit-exactness.
scripts/emu_sanitize.sh runs this file under ThreadSanitizer (shared-memory races) and
AddressSanitizer (out-of-bounds accesses)."""
import ctypes as C

import pytest
import torch

from oracle import costvolume_oracle as O
from simplerecon_b200 import _native as N
from simplerecon_b200.synthetic import make_tuple, mlp_state
from tests import emu
from tests.parity import (assert_cost_close, assert_lowest_close, assert_mask_close, golden_names,
                          load_golden)


@pytest.fixture(scope="module")
def lib():
    lib = emu.load_or_skip()
    yield lib
    lib.emu_set_sms(4)
    lib.srcv_set_variant(N.VARIANT_AUTO)


def _weights(K, C, hidden=(128, 128), seed=1):
    sd = mlp_state(views=K, channels=C, hidden=hidden, seed=seed)
    return [sd[f"mlp.net.{i}.{n}"].clone() for i in (0, 2, 4) for n in ("weight", "bias")]


def _rel(a, b):
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


# ----------------------------------------------------------------------------------------- #
# golden vectors of the unmodified reference (tests/golden), through the emulated C ABI       #
# ----------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("variant", ["generic", "auto"])
@pytest.mark.parametrize("name", golden_names())
def test_golden_through_emulated_abi(lib, name, variant):
    """Same check as tests/test_gpu_parity.py::test_golden, on the host-compiled kernel sources:
    reference fp32 / fp64 outputs, argmax depth and mask of every committed fixture."""
    g, inputs, sd = load_golden(name)
    kind, D = g["kind"], g["D"]
    C_ = inputs["src_feats"].shape[2]
    K_ = inputs["src_feats"].shape[1]
    if variant == "auto" and (C_ != 16 or (kind == "mlp" and K_ != 7)):
        pytest.skip("no second variant for this shape")
    lib.emu_set_sms(148 if variant == "auto" else 4)          # auto: exercise the plane-loop split
    lib.srcv_set_variant(N.VARIANT_GENERIC if variant == "generic" else N.VARIANT_AUTO)
    planes_in = inputs.get("depth_planes_bdhw")
    B, H, W = inputs["src_feats"].shape[0], inputs["src_feats"].shape[3], inputs["src_feats"].shape[4]
    if kind == "dot":
        cost, lowest, planes_bd, used = emu.dot_forward(inputs, D, planes=planes_in)
        mask = None
    else:
        wts = O.mlp_weights_from_state_dict(sd)
        cost, lowest, planes_bd, mask, used = emu.mlp_forward(inputs, D, wts, planes=planes_in)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    assert (("fast" in used) or ("wgmma" in used)) == (variant == "auto"), used
    assert_cost_close(kind, cost, g["ref_cost"], g["ref_cost64"], what=f"emu {name}/{used}")
    planes = planes_in if planes_in is not None else planes_bd.view(B, D, 1, 1)
    if planes_in is None:
        assert torch.allclose(planes_bd, g["ref_planes"], rtol=3e-7, atol=0)
    assert_lowest_close(kind, lowest, planes, g["ref_cost"], what=f"emu {name}")
    if kind == "mlp":
        assert_mask_close(mask, g["ref_mask"], what=f"emu {name}")


# ----------------------------------------------------------------------------------------- #
# dot-product sweep                                                                          #
# ----------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("B,K,C,H,W,D,sms,variant,expect", [
    (1, 2, 8, 10, 12, 5, 4, N.VARIANT_AUTO, "dot_generic"),            # C != 16: planar scalar gathers
    (2, 3, 16, 12, 16, 16, 4, N.VARIANT_AUTO, "dot_fast_c4planar"),    # plane loop not split: argmax in the sweep
    (2, 3, 16, 12, 16, 16, 148, N.VARIANT_AUTO, "dot_fast_c4planar"),  # split x2: last-arriver argmax
    (1, 2, 16, 9, 21, 32, 148, N.VARIANT_AUTO, "dot_fast_c4planar"),   # split x4, ragged tiles, HW % 4 != 0
    (1, 1, 16, 6, 40, 7, 4, N.VARIANT_AUTO, "dot_fast_c4planar"),      # one view, D not a multiple of the plane chunk
    (1, 2, 16, 12, 16, 6, 4, N.VARIANT_GENERIC, "dot_generic"),        # forced generic on a fast-capable shape
])
def test_dot_forward(lib, B, K, C, H, W, D, sms, variant, expect):
    lib.emu_set_sms(sms)
    lib.srcv_set_variant(variant)
    t = make_tuple(B, K, H, W, channels=C, seed=11 + D)
    cost, lowest, planes_bd, used = emu.dot_forward(t, D)
    assert used == expect
    oc, ol, op, _ = O.forward_dot(**t, num_depth_bins=D)
    assert_cost_close("dot", cost, oc, what=f"emu {used}")
    assert_lowest_close("dot", lowest, planes_bd.view(B, D, 1, 1), oc, what=f"emu {used}")
    assert _rel(planes_bd, op[:, :, 0, 0]) < 1e-6
    # the argmax is exactly the argmax of the kernel's own volume (fused / last-arriver / separate launch)
    idx = cost.argmax(1, keepdim=True)
    assert torch.equal(torch.gather(planes_bd.view(B, D, 1, 1).expand_as(cost), 1, idx).squeeze(1), lowest)


def test_dot_millimetre_depths_keep_the_reference_epsilon(lib):
    """Regression for a fuzzer finding: the reference divides by z' = z + 1e-8
    (utils/geometry_utils.py:83-87); in centred coordinates the numerator must carry -cxo*eps as
    well, otherwise the sample position is off by cxo*eps/z — 5e-5 px at z = 1 mm.  Judged
    against the fp64 evaluation like tests/parity.py."""
    lib.emu_set_sms(4)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    B, K, C_, H, W, D = 2, 4, 16, 6, 22, 4
    t = make_tuple(B, K, H, W, channels=C_, seed=77, t_range=(0.0, 0.0), max_angle=0.6)   # pure rotations
    t["min_depth"], t["max_depth"] = torch.full((1, 1, 1, 1), 1e-3), torch.full((1, 1, 1, 1), 1e-2)
    cost, _, _, used = emu.dot_forward(t, D)
    oc, *_ = O.forward_dot(**t, num_depth_bins=D)
    o64, *_ = O.forward_dot(**{k: v.double() for k, v in t.items()}, num_depth_bins=D)
    e_ref = (oc.double() - o64).abs().max().item()
    e_ours = (cost.double() - o64).abs().max().item()
    assert e_ours <= 2 * e_ref + 1e-6 * o64.abs().max().item(), (e_ours, e_ref, used)


@pytest.mark.parametrize("C,sms", [(8, 4), (16, 4), (16, 148)])
def test_dot_forward_per_pixel_planes(lib, C, sms):
    lib.emu_set_sms(sms)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    B, K, H, W, D = 1, 2, 10, 14, 16
    t = make_tuple(B, K, H, W, channels=C, seed=5)
    planes = 0.3 + 4.0 * torch.rand(B, D, H, W, generator=torch.Generator().manual_seed(6))
    cost, lowest, _, used = emu.dot_forward(t, D, planes=planes)
    oc, ol, _, _ = O.forward_dot(**t, num_depth_bins=D, depth_planes_bdhw=planes)
    assert_cost_close("dot", cost, oc, what=f"emu per-pixel {used}")
    assert_lowest_close("dot", lowest, planes, oc, what=f"emu per-pixel {used}")


@pytest.mark.parametrize("B,K,C,H,W,D,per_pixel", [(2, 3, 16, 10, 12, 5, False), (1, 2, 8, 9, 11, 4, True)])
def test_dot_backward(lib, B, K, C, H, W, D, per_pixel):
    t = make_tuple(B, K, H, W, channels=C, seed=71)
    g = torch.Generator().manual_seed(72)
    gcost = torch.randn(B, D, H, W, generator=g)
    planes = (0.3 + 4.0 * torch.rand(B, D, H, W, generator=g)) if per_pixel else None
    tc = dict(t)
    tc["cur_feats"] = t["cur_feats"].clone().requires_grad_(True)
    tc["src_feats"] = t["src_feats"].clone().requires_grad_(True)
    oc, _, op, _ = O.forward_dot(**tc, num_depth_bins=D, depth_planes_bdhw=planes)
    (oc * gcost).sum().backward()
    gcur, gsrc = emu.dot_backward(t, D, gcost, planes=planes if per_pixel else op[:, :, 0, 0].detach())
    assert _rel(gcur, tc["cur_feats"].grad) < 5e-5
    assert _rel(gsrc, tc["src_feats"].grad) < 5e-5


def test_warp_features(lib):
    B, K, C, H, W = 2, 3, 8, 9, 13
    t = make_tuple(B, K, H, W, channels=C, seed=41)
    plane = torch.tensor([1.3, 2.1])
    warped, depths, mask = emu.warp_features(t, plane, per_pixel=False)
    X = plane.view(B, 1, 1) * O.backproject_rays(t["cur_invK"], H, W)
    px, py, zp = O.project(X, t["src_Ks"], t["src_extrinsics"])
    ref = O.sample_bilinear_zeros(t["src_feats"], px, py).reshape(B, K, C, H, W)
    assert (warped - ref).abs().max().item() <= 4e-5 * ref.abs().max().item() + 1e-6
    assert _rel(depths, zp.reshape(B, K, H, W)) < 1e-5
    assert ((mask > 0.5) != (zp.reshape(B, K, H, W) > 0)).float().mean().item() < 1e-3


# ----------------------------------------------------------------------------------------- #
# metadata-MLP sweep (fp32 SIMT variant) and its backward                                     #
# ----------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("B,K,C,H,W,D,hidden,per_pixel", [
    (1, 2, 8, 10, 12, 3, (128, 128), False),
    (1, 7, 16, 8, 9, 2, (128, 128), False),       # hero channel count (202), ragged last tile
    (2, 3, 16, 9, 11, 2, (96, 64), True),
])
def test_mlp_forward(lib, B, K, C, H, W, D, hidden, per_pixel):
    lib.srcv_set_variant(N.VARIANT_GENERIC)         # the fp32 SIMT variant (the hero layout would pick wgmma)
    t = make_tuple(B, K, H, W, channels=C, seed=21)
    wts = _weights(K, C, hidden)
    planes = (0.3 + 4.0 * torch.rand(B, D, H, W, generator=torch.Generator().manual_seed(22))) if per_pixel else None
    cost, lowest, planes_bd, mask, used = emu.mlp_forward(t, D, wts, planes=planes)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    assert used == "mlp_generic_fp32"
    oc, ol, op, om = O.forward_mlp(**t, weights=tuple(wts), num_depth_bins=D, depth_planes_bdhw=planes,
                                   return_mask=True)
    assert_cost_close("mlp", cost, oc, what="emu mlp_generic")
    assert_lowest_close("mlp", lowest, planes if per_pixel else planes_bd.view(B, D, 1, 1), oc, what="emu mlp_generic")
    assert_mask_close(mask, om, what="emu mlp_generic")


@pytest.mark.parametrize("B,K,C,H,W,D,hidden,per_pixel,sms", [
    (1, 2, 8, 10, 12, 3, (128, 128), False, 2),    # F = 48 -> 64-wide feature tile; CTAs loop over tiles
    (1, 7, 16, 8, 8, 2, (128, 128), False, 4),     # hero layout: F = 202 -> 208
    (2, 3, 16, 9, 11, 2, (96, 64), True, 3),       # F = 98 -> 128; narrow hidden layers; ragged tiles
])
def test_mlp_backward(lib, B, K, C, H, W, D, hidden, per_pixel, sms):
    """srcv_mlp_backward_f32 against autograd through the oracle (the composite the reference
    differentiates, modules/cost_volume.py:451-736 + modules/networks.py:129-147)."""
    lib.emu_set_sms(sms)
    t = make_tuple(B, K, H, W, channels=C, seed=3)
    wts = _weights(K, C, hidden)
    g = torch.Generator().manual_seed(4)
    gcost = torch.randn(B, D, H, W, generator=g)
    planes = (0.3 + 4.0 * torch.rand(B, D, H, W, generator=g)) if per_pixel else None
    # fp64 oracle gradients: the fp32 composite flips LeakyReLU kinks (a ~1e-7 pre-activation) more
    # often than the kernel does, see scripts/emu_fuzz.py
    tc = {k: v.double() for k, v in t.items()}
    tc["cur_feats"] = tc["cur_feats"].clone().requires_grad_(True)
    tc["src_feats"] = tc["src_feats"].clone().requires_grad_(True)
    wo = [w.double().clone().requires_grad_(True) for w in wts]
    oc, _, op, _ = O.forward_mlp(**tc, weights=tuple(wo), num_depth_bins=D,
                                 depth_planes_bdhw=None if planes is None else planes.double())
    (oc * gcost.double()).sum().backward()
    ref = [tc["cur_feats"].grad, tc["src_feats"].grad] + [w.grad for w in wo]
    op = op.float()
    ours = emu.mlp_backward(t, D, wts, gcost, planes=planes if per_pixel else op[:, :, 0, 0].detach())
    for name, o, r in zip(("cur", "src", "w1", "b1", "w2", "b2", "w3", "b3"), ours, ref):
        assert o.shape == r.shape
        assert _rel(o.double(), r) < 2e-5, f"grad {name}: rel err {_rel(o.double(), r):.2e}"


# ----------------------------------------------------------------------------------------- #
# wgmma kernel against the functional wgmma / mbarrier model (tests/emu/emu_tc.h)       #
# ----------------------------------------------------------------------------------------- #
def test_tc_selftest_three_product_gemm(lib):
    """srcv_tc_selftest_f32: D = A W^T through wgmma with the (hi, lo) fp16 split."""
    g = torch.Generator().manual_seed(0)
    for Kp, scale in ((64, 0.1), (208, 1.0)):
        A, Wm = torch.randn(128, Kp, generator=g), scale * torch.randn(128, Kp, generator=g)
        Dm = torch.full((128, 128), float("nan"))
        scratch = torch.zeros(2 * 128 * Kp * 2 + 256, dtype=torch.uint8)
        assert lib.srcv_tc_selftest_f32(emu._p(A), emu._p(Wm), Kp, emu._p(Dm), emu._p(scratch), None) == 0
        ref = A.double() @ Wm.double().T
        assert (Dm.double() - ref).abs().max().item() <= 4e-6 * ref.abs().max().item()
    assert lib.srcv_tc_selftest_f32(emu._p(A), emu._p(Wm), 40, emu._p(Dm), emu._p(scratch), None) != 0   # Kp % 16


@pytest.mark.parametrize("B,H,W,D,per_pixel,sms", [
    (1, 8, 16, 8, False, 2),      # 16 tiles over 2 persistent CTAs: the steady-state pipeline (prologue, overlap, drain)
    (2, 5, 19, 6, False, 3),      # ragged patches (partial 16x2 tiles), 2 frames
    (2, 5, 19, 5, False, 3),      # ... and D not a multiple of the 2-plane tile
    (1, 6, 16, 4, True, 8),       # per-pixel planes; more CTAs than tiles per CTA > 1
])
def test_mlp_forward_wgmma(lib, B, H, W, D, per_pixel, sms):
    """mlp_tc_kernel (K = 7, C = 16, 128/128): 512 host threads per CTA run the real builder / consumer-warpgroup
    code; wgmma (executed at issue), mbarriers and the bulk copy are the functional
    model.  Checks the protocol (no deadlock, no lost tile) and the arithmetic against the oracle."""
    lib.emu_set_sms(sms)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    K, C_ = 7, 16
    t = make_tuple(B, K, H, W, channels=C_, seed=51)
    wts = _weights(K, C_)
    planes = (0.3 + 4.0 * torch.rand(B, D, H, W, generator=torch.Generator().manual_seed(52))) if per_pixel else None
    cost, lowest, planes_bd, mask, used = emu.mlp_forward(t, D, wts, planes=planes)
    assert used == "mlp_tc_wgmma_f16x3"
    oc, ol, op, om = O.forward_mlp(**t, weights=tuple(wts), num_depth_bins=D, depth_planes_bdhw=planes,
                                   return_mask=True)
    assert_cost_close("mlp", cost, oc, what="emu wgmma")
    assert_lowest_close("mlp", lowest, planes if per_pixel else planes_bd.view(B, D, 1, 1), oc, what="emu wgmma")
    assert_mask_close(mask, om, what="emu wgmma")
    # the fp32 SIMT variant of the same call agrees to the split's 2^-21
    lib.srcv_set_variant(N.VARIANT_GENERIC)
    cost_g, *_ = emu.mlp_forward(t, D, wts, planes=planes)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    assert (cost - cost_g).abs().max().item() <= 2e-5 * oc.abs().max().item() + 1e-6


def test_dot_forward_compile_time_map_size(lib):
    """The 160x120 instantiation of the fast dot sweep (compile-time tap offsets) — the kernel the
    BASELINE configs run — on one full-size frame with few planes."""
    lib.emu_set_sms(4)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    B, K, C_, H, W, D = 1, 2, 16, 120, 160, 8
    t = make_tuple(B, K, H, W, channels=C_, seed=91)
    cost, lowest, planes_bd, used = emu.dot_forward(t, D)
    assert used == "dot_fast_c4planar"
    oc, *_ = O.forward_dot(**t, num_depth_bins=D)
    assert_cost_close("dot", cost, oc, what="emu dot 160x120")
    assert_lowest_close("dot", lowest, planes_bd.view(B, D, 1, 1), oc, what="emu dot 160x120")


@pytest.mark.skipif(not __import__("os").environ.get("SRCV_EMU_SLOW"), reason="several minutes: set SRCV_EMU_SLOW=1")
def test_mlp_forward_wgmma_compile_time_map_size(lib):
    """The 160x120 instantiation of the wgmma kernel on one full-size frame, one plane chunk
    (600 tiles through the 640-thread pipeline)."""
    lib.emu_set_sms(8)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    B, K, C_, H, W, D = 1, 7, 16, 120, 160, 4
    t = make_tuple(B, K, H, W, channels=C_, seed=92)
    wts = _weights(K, C_)
    cost, lowest, planes_bd, mask, used = emu.mlp_forward(t, D, wts)
    assert used == "mlp_tc_wgmma_f16x3"
    oc, ol, op, om = O.forward_mlp(**t, weights=tuple(wts), num_depth_bins=D, return_mask=True)
    o64, *_ = O.forward_mlp(**{k: v.double() for k, v in t.items()}, weights=tuple(w.double() for w in wts),
                            num_depth_bins=D)
    # at 160-pixel coordinates the reference's own fp32 run is ~1.5e-5 off its fp64 evaluation
    assert_cost_close("mlp", cost, oc, o64, what="emu wgmma 160x120")
    assert_mask_close(mask, om, what="emu wgmma 160x120")


def test_forward_sweeps_are_deterministic(lib):
    """The forward kernels have no order-dependent arithmetic (the split dot sweep reduces through
    the last-arriver, the hero kernel reduces its four quarters in a fixed order): two runs with
    differently interleaved host threads must agree bit for bit."""
    lib.emu_set_sms(148)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    t = make_tuple(1, 7, 8, 16, channels=16, seed=61)
    a = emu.dot_forward(t, 16)
    b = emu.dot_forward(t, 16)
    assert a[3] == "dot_fast_c4planar" and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    lib.emu_set_sms(3)
    wts = _weights(7, 16)
    a = emu.mlp_forward(t, 8, wts)
    b = emu.mlp_forward(t, 8, wts)
    assert a[4] == "mlp_tc_wgmma_f16x3"
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])


# ----------------------------------------------------------------------------------------- #
# C-ABI argument validation (srcv_api.cu) — runs the real front end, no kernel is launched    #
# ----------------------------------------------------------------------------------------- #
def test_api_validation(lib):
    t = make_tuple(1, 2, 8, 10, channels=16, seed=1)
    c = emu.Call(t, 4)
    cost, lowest = torch.empty(1, 4, 8, 10), torch.empty(1, 8, 10)
    n = lib.srcv_dot_workspace_bytes(C.byref(c.shape))
    ws = c.workspace(n)
    p = emu._p

    def call(shape=c.shape, cur=t["cur_feats"], ws_=ws, nbytes=n, pl=c.pl, cams=c.cams):
        return lib.srcv_dot_forward_f32(C.byref(shape), p(cur), p(c.t["src_feats"]), C.byref(cams), C.byref(pl),
                                        p(cost), p(lowest), p(ws_), nbytes, None)

    assert call() == 0
    assert call(nbytes=n - 1) != 0 and b"workspace too small" in lib.srcv_last_error()
    assert call(ws_=ws[16:]) != 0 and b"256-byte aligned" in lib.srcv_last_error()
    assert call(cur=None) != 0
    assert call(shape=N.Shape(1, 2, 16, 8, 0, 4)) != 0 and b"non-positive" in lib.srcv_last_error()
    bad = N.Planes()
    bad.mode = 9
    assert call(pl=bad) != 0 and b"unknown planes mode" in lib.srcv_last_error()
    assert call(cams=N.Cameras(None, None, None, None)) != 0
    # unaligned feature pointer (the kernels use 16-byte vector loads)
    assert call(cur=c.t["cur_feats"].reshape(-1)[1:]) != 0 and b"16-byte aligned" in lib.srcv_last_error()
    # forcing the fast variant on a shape it does not support is an error, not a silent fallback
    t8 = make_tuple(1, 2, 8, 10, channels=8, seed=2)
    lib.srcv_set_variant(N.VARIANT_FAST)
    with pytest.raises(N.SrcvError):
        emu.dot_forward(t8, 4)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    assert lib.srcv_set_variant(77) != 0
    # MLP: hidden widths beyond the build, inconsistent workspace query
    w = N.MlpWeights(1, 1, 1, 1, 1, 1, 256, 128)
    assert lib.srcv_mlp_workspace_bytes(C.byref(c.shape), C.byref(w)) == 0
    assert lib.srcv_mlp_backward_workspace_bytes(C.byref(N.Shape(1, 12, 16, 8, 10, 4)),
                                                 C.byref(N.MlpWeights(1, 1, 1, 1, 1, 1, 128, 128))) == 0   # F = 332 > 208
