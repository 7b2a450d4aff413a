"""CPU: the normals kernels (csrc/srcv_normals.cuh) compiled for the host (tests/emu) behind the Python mirrors of
the reference's NormalGenerator and NormalsLoss, against the fp64 oracle (oracle/normals_oracle.py):
normals, the depth gradient, the loss and both of its gradients, the C ABI's argument checks, the state_dict
keys, install()/uninstall() and the launch counts."""
import contextlib
import ctypes as C
import types

import pytest
import torch

from oracle import normals_oracle as O
from oracle.ref_import import reference_available
from simplerecon_b200 import _native, normals as NM
from simplerecon_b200.synthetic import make_normals_batch
from tests import emu


@pytest.fixture()
def emulated(monkeypatch):
    lib = emu.load_or_skip()
    monkeypatch.setattr(_native, "_lib", lib)
    monkeypatch.setattr(NM, "_require_cuda", lambda t: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: types.SimpleNamespace(cuda_stream=0))
    real_empty = torch.empty

    def aligned_empty(*size, **kw):
        if kw.get("dtype") is torch.uint8 and len(size) == 1 and isinstance(size[0], int):
            buf = real_empty(size[0] + 256, **kw)
            off = (-buf.data_ptr()) % 256
            return buf[off:off + size[0]]
        return real_empty(*size, **kw)

    monkeypatch.setattr(torch, "empty", aligned_empty)
    return lib


# (seed, B, H, W): the shapes of the stored reference outputs, then 17x23 and 48x64
SHAPES = [(0, 3, 24, 32), (1, 1, 17, 23), (2, 1, 3, 3), (3, 3, 5, 4), (4, 1, 9, 31), (5, 2, 48, 64)]
KERNELS = [(5, 2.0), (3, 1.0), (7, 3.0)]


def check_normals(depth, invK, k=5, sigma=2.0, device="cpu"):
    """normals of the mirror against the fp64 oracle: the same all-finite mask, and
    max|n - n64| <= 2 max|n32 - n64| + 1e-6 over the finite pixels (n32 = the fp32 oracle)"""
    ng = NM.NormalGenerator(depth.shape[-2], depth.shape[-1], k, sigma).to(device)
    n = ng(depth.to(device), invK.to(device)).cpu()
    n32 = O.normal_generator(depth, invK, k, sigma)
    n64 = O.normal_generator(depth.double(), invK.double(), k, sigma)
    fin = O.all_finite(n)
    assert torch.equal(fin, O.all_finite(n64)) and torch.equal(fin, O.all_finite(n32))
    assert torch.isnan(n.permute(1, 0, 2, 3)[:, ~fin]).all()           # all three components NaN
    m = fin[:, None].expand_as(n)
    if not m.any():
        return n
    err, err32 = (n.double() - n64)[m].abs().max().item(), (n32.double() - n64)[m].abs().max().item()
    assert err <= 2 * err32 + 1e-6, (err, err32)
    return n


def check_depth_gradient(depth, invK, k=5, sigma=2.0, device="cpu", seed=0):
    """d sum(n . g_n) / d depth against fp64 autograd through the oracle: within 1e-4 of max|g64| where the
    oracle's gradient is finite (a non-finite depth in a window makes the reference's NaN); finite everywhere"""
    g_n = torch.randn(depth.shape[0], 3, *depth.shape[-2:], generator=torch.Generator().manual_seed(seed))
    n64 = O.normal_generator(depth.double(), invK.double(), k, sigma)
    g_n[~O.all_finite(n64)[:, None].expand_as(g_n)] = 0.0               # as NormalsLoss masks them
    d = depth.to(device).clone().requires_grad_(True)
    ng = NM.NormalGenerator(depth.shape[-2], depth.shape[-1], k, sigma).to(device)
    (ng(d, invK.to(device)) * g_n.to(device)).sum().backward()
    d64 = depth.double().clone().requires_grad_(True)
    (O.normal_generator(d64, invK.double(), k, sigma) * g_n.double()).sum().backward()
    g, g64 = d.grad.cpu().double(), d64.grad
    assert torch.isfinite(g).all()
    ok = torch.isfinite(g64)
    if not ok.any():                                                   # a tiny map entirely under a hole
        return g
    scale = g64[ok].abs().max()
    assert scale > 0
    err = (g - g64)[ok].abs().max()
    assert err <= 1e-4 * scale, (err.item(), scale.item())
    return g


def check_loss(gt_n, pred_n, device="cpu"):
    """loss within 2e-5 relative of the fp64 oracle, both gradients against fp64 autograd"""
    a = gt_n.to(device).clone().requires_grad_(True)
    b = pred_n.to(device).clone().requires_grad_(True)
    loss = NM.NormalsLoss()(a, b)
    loss.backward()
    a64, b64 = gt_n.double().clone().requires_grad_(True), pred_n.double().clone().requires_grad_(True)
    l64 = O.normals_loss(a64, b64)
    l64.backward()
    assert loss.dtype == torch.float32 and loss.shape == ()
    if torch.isnan(l64):                                               # no pixel in the mask
        assert torch.isnan(loss) and not a.grad.any() and not b.grad.any()
        return loss
    assert abs(loss.item() - l64.item()) <= 2e-5 * abs(l64.item()) + 1e-7, (loss.item(), l64.item())
    for g, g64 in ((a.grad, a64.grad), (b.grad, b64.grad)):
        assert torch.isfinite(g).all() and torch.isfinite(g64).all()
        assert (g.cpu().double() - g64).abs().max() <= 1e-5 * g64.abs().max() + 1e-12
    return loss


def _batch(seed, B, H, W, holes=True):
    t = make_normals_batch(seed, B, H, W, holes=holes)
    return t["depth_gt_b1hw"], t["depth_pred_b1hw"], t["invK_b44"]


@pytest.mark.parametrize("k,sigma", KERNELS)
@pytest.mark.parametrize("seed,B,H,W", SHAPES)
def test_normals_forward(emulated, seed, B, H, W, k, sigma):
    if min(H, W) <= k // 2:
        pytest.skip("below the reflect padding's minimum size")
    gt, pred, invK = _batch(seed, B, H, W)
    n = check_normals(gt, invK, k, sigma)
    if min(H, W) > 4:
        assert (~O.all_finite(n)).any()                                 # the holes reach the output
    check_normals(pred, invK, k, sigma)


@pytest.mark.parametrize("k,sigma", KERNELS)
@pytest.mark.parametrize("seed,B,H,W", SHAPES)
def test_depth_gradient(emulated, seed, B, H, W, k, sigma):
    if min(H, W) <= k // 2:
        pytest.skip("below the reflect padding's minimum size")
    gt, pred, invK = _batch(seed, B, H, W)
    check_depth_gradient(pred, invK, k, sigma, seed=seed)
    holes = torch.where(torch.isnan(gt), gt, pred)                    # NaN holes, no zero patch
    check_depth_gradient(holes, invK, k, sigma, seed=seed + 1)


def test_fronto_parallel_plane(emulated):
    K = torch.eye(4)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = 128.0, 64.0, 16.5, 11.25
    invK = torch.inverse(K)[None].repeat(2, 1, 1)
    n = NM.NormalGenerator(19, 37)(torch.full((2, 1, 19, 37), 2.0), invK)
    assert torch.all((n[:, :2].abs() <= 1e-6) & ((n[:, 2] - 1).abs() <= 1e-6))


@pytest.mark.parametrize("seed,B,H,W", SHAPES)
def test_loss_and_gradients(emulated, seed, B, H, W):
    gt, pred, invK = _batch(seed, B, H, W)
    gt_n, pred_n = O.normal_generator(gt, invK), O.normal_generator(pred, invK)
    check_loss(gt_n, pred_n)


def test_training_step_composition(emulated):
    """NormalsLoss(NG(gt), NG(pred)) and its gradient w.r.t. the predicted depth (depth_model.py:526-530, :475)"""
    gt, pred, invK = _batch(7, 2, 30, 40)
    ng, crit = NM.NormalGenerator(30, 40), NM.NormalsLoss()
    p = pred.clone().requires_grad_(True)
    loss = crit(ng(gt, invK), ng(p, invK))
    loss.backward()
    p64 = pred.double().clone().requires_grad_(True)
    l64 = O.normals_loss(O.normal_generator(gt.double(), invK.double()), O.normal_generator(p64, invK.double()))
    l64.backward()
    assert abs(loss.item() - l64.item()) <= 2e-5 * l64.item()
    assert torch.isfinite(p.grad).all() and torch.isfinite(p64.grad).all()
    assert (p.grad.double() - p64.grad).abs().max() <= 1e-4 * p64.grad.abs().max()


def test_empty_mask_gives_nan_and_zero_gradients(emulated):
    gt_n = torch.full((2, 3, 6, 7), float("nan"))
    pred_n = torch.randn(2, 3, 6, 7).requires_grad_(True)
    a = gt_n.clone().requires_grad_(True)
    loss = NM.NormalsLoss()(a, pred_n)
    assert torch.isnan(loss)
    loss.backward()
    assert torch.equal(pred_n.grad, torch.zeros_like(pred_n)) and torch.equal(a.grad, torch.zeros_like(a))
    assert torch.isnan(O.normals_loss(gt_n, pred_n.detach()))


def test_half_inputs_are_upcast(emulated):
    gt, pred, invK = _batch(8, 1, 16, 20, holes=False)
    ph = pred.half().requires_grad_(True)
    n = NM.NormalGenerator(16, 20)(ph, invK)
    assert n.dtype == torch.float16
    n64 = O.normal_generator(ph.detach().double(), invK.double())
    assert (n.double() - n64).abs().max() <= 2e-3                     # fp32 result rounded to fp16
    n.float().sum().backward()
    assert ph.grad.dtype == torch.float16 and torch.isfinite(ph.grad).all()


def _args(depth, invK, taps, k, B=None, H=None, W=None):
    return _native.NormalsArgs(depth.data_ptr(), invK.data_ptr(), taps.data_ptr(), B or depth.shape[0],
                               H or depth.shape[-2], W or depth.shape[-1], k)


def test_argument_checks(emulated):
    lib = emulated
    depth, invK, taps = torch.rand(1, 1, 8, 9) + 1, torch.eye(4)[None], NM.gaussian_taps(5, 2.0)
    out = torch.empty(1, 3, 8, 9)
    for k, H in ((4, 8), (17, 8), (0, 8), (5, 2), (7, 3)):
        a = _args(depth, invK, taps, k, H=H)
        assert lib.srcv_normals_forward_f32(C.byref(a), C.c_void_p(out.data_ptr()), None) == 2
        assert lib.srcv_normals_workspace_bytes(C.byref(a)) == 0
    a = _args(depth, invK, taps, 5)
    assert lib.srcv_normals_forward_f32(C.byref(a), None, None) == 1
    assert lib.srcv_normals_forward_f32(C.byref(_args(depth, invK, taps, 5, B=70000)), C.c_void_p(out.data_ptr()),
                                        None) == 2
    n = lib.srcv_normals_workspace_bytes(C.byref(a))
    assert n >= 24 * 8 * 9
    g = torch.zeros(1, 3, 8, 9)
    assert lib.srcv_normals_backward_f32(C.byref(a), C.c_void_p(g.data_ptr()), C.c_void_p(out.data_ptr()),
                                         None, 0, None) == 1
    assert lib.srcv_normals_loss_forward_f32(C.c_void_p(out.data_ptr()), C.c_void_p(out.data_ptr()), 0, 8, 9,
                                             C.c_void_p(out.data_ptr()), None, 0, None) == 2
    assert lib.srcv_normals_loss_workspace_bytes(1, 0, 9) == 0
    ng = NM.NormalGenerator(8, 9)
    with pytest.raises(ValueError):
        ng(torch.rand(1, 1, 8, 10), invK)                              # not the constructor's (H, W)
    with pytest.raises(ValueError):
        ng(depth, torch.eye(4)[None].repeat(2, 1, 1))
    with pytest.raises(_native.SrcvError):
        NM.NormalGenerator(2, 9)(torch.rand(1, 1, 2, 9), invK)         # H <= k // 2
    with pytest.raises(ValueError):
        NM.NormalsLoss()(torch.rand(1, 3, 4, 4), torch.rand(1, 3, 4, 5))


def test_launch_counts_and_determinism(emulated):
    gt, pred, invK = _batch(9, 2, 20, 36)
    ng, crit = NM.NormalGenerator(20, 36), NM.NormalsLoss()
    runs = []
    for _ in range(2):
        p = pred.clone().requires_grad_(True)
        c0 = _native.launch_count()
        n_gt = ng(gt, invK)
        c1 = _native.launch_count()
        n_p = ng(p, invK)
        loss = crit(n_gt, n_p)
        c2 = _native.launch_count()
        loss.backward()
        c3 = _native.launch_count()
        assert (c1 - c0, c2 - c1, c3 - c2) == (1, 1 + 2, 1 + 2)       # NG; NG + loss; loss + NG backward
        runs.append((n_gt, n_p, loss, p.grad))
    for x, y in zip(*runs):
        assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))


REFERENCE_KEYS = ["backproject.pix_coords_13N"]


def test_state_dict_matches_the_reference():
    ours = NM.NormalGenerator(12, 16).state_dict()
    assert list(ours) == REFERENCE_KEYS
    assert torch.equal(ours["backproject.pix_coords_13N"], O.pix_coords(12, 16))
    assert list(NM.NormalsLoss().state_dict()) == []
    if reference_available():
        ref = O.load_reference_normals().NormalGenerator(12, 16)
        assert list(ref.state_dict()) == REFERENCE_KEYS
        assert torch.equal(ref.state_dict()["backproject.pix_coords_13N"], ours["backproject.pix_coords_13N"])
        NM.NormalGenerator(12, 16).load_state_dict(ref.state_dict(), strict=True)


@pytest.mark.skipif(not reference_available(), reason="needs $SIMPLERECON_REF (the reference tree)")
def test_install_and_uninstall_on_the_reference_modules():
    from simplerecon_b200 import install, uninstall
    ref = O.load_reference_normals()
    geo, losses = ref.geometry, ref.losses
    orig = (geo.NormalGenerator, losses.NormalsLoss, losses.MVDepthLoss)
    try:
        install(normals=True)
        assert geo.NormalGenerator is NM.NormalGenerator and losses.NormalsLoss is NM.NormalsLoss
        assert losses.MVDepthLoss is orig[2]                           # other flags keep their behaviour
    finally:
        uninstall()
    assert (geo.NormalGenerator, losses.NormalsLoss, losses.MVDepthLoss) == orig
