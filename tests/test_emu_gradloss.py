"""CPU: the gradient-loss kernels (csrc/srcv_gradloss.cuh) compiled for the host (tests/emu) behind the Python mirrors
of the reference's MSGradientLoss and ScaleInvariantLoss, against the fp64 oracle (oracle/gradloss_oracle.py): the
loss, the per-level mask counts, the gradient to the prediction, the C ABI's argument checks, the empty state_dict,
install()/uninstall() and the launch counts."""
import contextlib
import ctypes as C
import sys
import types

import pytest
import torch

import simplerecon_b200 as S
from oracle import gradloss_oracle as O
from oracle.normals_oracle import spatial_gradient
from simplerecon_b200 import _native, losses as L
from simplerecon_b200.synthetic import make_normals_batch
from tests import emu


@pytest.fixture()
def emulated(monkeypatch):
    lib = emu.load_or_skip()
    monkeypatch.setattr(_native, "_lib", lib)
    monkeypatch.setattr(L, "_require_cuda", lambda t: None)
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


# (seed, B, H, W): the shapes of the stored reference outputs, then 3x3 (levels 3, 2, 1, 1) and 5x4 (3x2, 2x1, 1x1)
SHAPES = [(0, 3, 24, 32), (1, 1, 17, 23), (3, 3, 5, 4), (2, 1, 3, 3), (4, 1, 9, 31), (5, 2, 48, 64)]


def near_zero_footprint(gt64, pred64, num_scales):
    """How many level-0 pixels a sign flip of a near-zero gradient difference can reach: for every masked
    component whose fp64 |delta| is within fp32 rounding of zero, the Sobel adjoint's 3x3 at its level, widened by
    each blur-pool adjoint on the way down (at most (4 * 2^l)^2 pixels)."""
    thr = 4e-6 * max(1.0, pred64.abs().max().item())
    total = 0
    for lvl, (p, g) in enumerate(zip(O.pyrdown(pred64, num_scales), O.pyrdown(gt64, num_scales))):
        gg = spatial_gradient(g)
        delta = spatial_gradient(p) - gg
        total += int((gg.isfinite() & (delta.abs() <= thr)).sum()) * (4 * 2 ** lvl) ** 2
    return total


def check_msgrad(gt, pred, num_scales=4, device="cpu"):
    """MSGradientLoss against the fp64 oracle:
      - |l - l64| <= 2 |l32 - l64| + 1e-6 |l64| + ulp (l32 = the fp32 oracle; ulp = 2^-24 max|depth|, what one
        fp32 rounding of a depth moves a term by: on a map of a few pixels l32 can land closer to l64 than
        fp32 terms warrant), NaN exactly when the oracle's is;
      - the workspace's per-level counts = the oracle's mask sums;
      - the gradient within 1e-4 of max|g64|, except at pixels a sign flip of a near-zero delta can reach, which
        are counted against `near_zero_footprint` (masks are compared by count, not by tolerance: DESIGN §2)."""
    p = pred.to(device).clone().requires_grad_(True)
    loss = L.MSGradientLoss(num_scales)(gt.to(device), p)
    assert loss.dtype == torch.float32 and loss.shape == () and loss.device == p.device
    loss.backward()
    assert p.grad.dtype == pred.dtype
    gt64, p64 = gt.double(), pred.double().clone().requires_grad_(True)
    l64 = O.ms_gradient_loss(gt64, p64, num_scales)
    l64.backward()
    l32 = O.ms_gradient_loss(gt.float(), pred.float(), num_scales)
    _, ws = L._msgrad_forward(gt.to(device).float().contiguous(), pred.to(device).float().contiguous(), num_scales)
    counts = ws[:32].cpu().view(torch.int64).tolist()
    want = [int(m.sum()) for m in O.level_masks(gt.float(), num_scales)]
    assert counts == want + [0] * (4 - num_scales)
    if torch.isnan(l64):
        assert torch.isnan(loss) and min(want) == 0
    else:
        err, err32 = abs(loss.item() - l64.item()), abs(l32.item() - l64.item())
        ulp = 2.0 ** -24 * pred.abs().max().item()
        assert err <= 2 * err32 + 1e-6 * abs(l64.item()) + ulp, (loss.item(), l64.item(), l32.item())
    g, g64 = p.grad.cpu().double(), p64.grad
    assert torch.isfinite(g).all() and torch.isfinite(g64).all()
    scale = g64.abs().max().item()
    # a half / bfloat16 gradient was rounded to that dtype: its relative step, and fp16's subnormal spacing (a mean
    # over 10^6 components puts the unscaled gradient below fp16's smallest normal)
    fi = torch.finfo(pred.dtype)
    half, spacing = (fi.eps, fi.smallest_normal * fi.eps) if pred.dtype != torch.float32 else (0.0, 0.0)
    bad = int(((g - g64).abs() > (1e-4 + half) * scale + spacing).sum())
    assert bad <= near_zero_footprint(gt64, p64.detach(), num_scales), (bad, scale)
    assert bad <= 0.01 * g.numel()
    return loss, p.grad


def check_si(gt, pred, si_lambda=0.85, device="cpu"):
    a, b = gt.to(device).clone().requires_grad_(True), pred.to(device).clone().requires_grad_(True)
    loss = L.ScaleInvariantLoss(si_lambda)(a, b)
    assert loss.dtype == torch.float32 and loss.shape == ()
    loss.backward()
    a64, b64 = gt.double().clone().requires_grad_(True), pred.double().clone().requires_grad_(True)
    l64 = O.scale_invariant_loss(a64, b64, si_lambda)
    l64.backward()
    if torch.isnan(l64):
        assert torch.isnan(loss)
        return loss
    assert abs(loss.item() - l64.item()) <= 2e-6 * abs(l64.item()), (loss.item(), l64.item())
    for g, g64 in ((a.grad, a64.grad), (b.grad, b64.grad)):
        assert g.shape == g64.shape
        assert (g.cpu().double() - g64).abs().max() <= 1e-5 * g64.abs().max()
    assert torch.equal(a.grad, -b.grad)
    return loss


def _batch(seed, B, H, W, holes=True):
    t = make_normals_batch(seed, B, H, W, holes=holes)
    return t["depth_gt_b1hw"], t["depth_pred_b1hw"]


@pytest.mark.parametrize("num_scales", [4, 3, 2, 1])
@pytest.mark.parametrize("seed,B,H,W", SHAPES)
def test_loss_counts_and_gradient(emulated, seed, B, H, W, num_scales):
    gt, pred = _batch(seed, B, H, W, holes=min(H, W) > 5)
    check_msgrad(gt, pred, num_scales)


def test_ground_truth_without_holes_and_an_all_nan_image(emulated):
    gt, pred = _batch(6, 2, 24, 32, holes=False)
    loss, _ = check_msgrad(gt, pred)
    assert torch.isfinite(loss)
    gt[1] = float("nan")                                               # the mask is over the whole batch
    loss, g = check_msgrad(gt, pred)
    assert torch.isfinite(loss) and not g[1].any() and g[0].any()


def test_an_empty_level_gives_nan_and_the_other_levels_gradient(emulated):
    gt, pred = _batch(0, 3, 24, 32)                                    # the holes cover the 3x4 level
    loss, g = check_msgrad(gt, pred)
    assert torch.isnan(loss) and g.any()
    loss, g = check_msgrad(torch.full((1, 1, 6, 7), float("nan")), torch.rand(1, 1, 6, 7))
    assert torch.isnan(loss) and not g.any()


def test_a_non_finite_prediction_inside_the_mask_gives_nan(emulated):
    gt, pred = _batch(6, 1, 12, 16, holes=False)
    pred[0, 0, 5, 5] = float("inf")
    p = pred.clone().requires_grad_(True)
    loss = L.MSGradientLoss()(gt, p)
    assert torch.isnan(loss) and torch.isnan(O.ms_gradient_loss(gt, pred))


def test_half_inputs_are_upcast(emulated):
    gt, pred = _batch(8, 1, 16, 20, holes=False)
    _, g = check_msgrad(gt.half(), pred.half())
    assert g.dtype == torch.float16
    _, g = check_msgrad(gt, pred.bfloat16())
    assert g.dtype == torch.bfloat16


@pytest.mark.parametrize("n", [1, 7, 100000])
def test_scale_invariant_loss(emulated, n):
    g = torch.Generator().manual_seed(n)
    gt = torch.randn(n, generator=g)
    pred = gt + 0.3 * torch.randn(n, generator=g) + 0.1
    check_si(gt, pred)
    if n == 7:
        check_si(gt.reshape(7, 1), pred.reshape(7, 1), si_lambda=0.5)
        assert torch.isnan(check_si(gt, gt - 1.0, si_lambda=1.5))      # negative radicand, as torch.sqrt


def test_scale_invariant_loss_of_an_empty_input(emulated):
    a, b = torch.empty(0, requires_grad=True), torch.empty(0, requires_grad=True)
    loss = L.ScaleInvariantLoss()(a, b)
    assert torch.isnan(loss)
    loss.backward()
    assert a.grad.shape == (0,) and b.grad.shape == (0,)


def test_argument_checks(emulated):
    lib = emulated
    x = torch.rand(1, 1, 8, 9)
    out = torch.empty(1)
    p = C.c_void_p(x.data_ptr())
    n = lib.srcv_msgrad_workspace_bytes(1, 8, 9, 4)
    ws = torch.empty(n, dtype=torch.uint8)
    w = C.c_void_p(ws.data_ptr())
    assert lib.srcv_msgrad_forward_f32(p, p, 1, 8, 9, 4, C.c_void_p(out.data_ptr()), w, n, None) == 0
    for B, H, W, s in ((1, 8, 9, 0), (1, 8, 9, 5), (70000, 8, 9, 4), (0, 8, 9, 4), (1, 0, 9, 4), (4, 1 << 14, 1 << 14, 4)):
        assert lib.srcv_msgrad_workspace_bytes(B, H, W, s) == 0
        assert lib.srcv_msgrad_forward_f32(p, p, B, H, W, s, C.c_void_p(out.data_ptr()), w, n, None) == 2
    assert lib.srcv_msgrad_forward_f32(None, p, 1, 8, 9, 4, C.c_void_p(out.data_ptr()), w, n, None) == 1
    assert lib.srcv_msgrad_forward_f32(p, p, 1, 8, 9, 4, None, w, n, None) == 1
    assert lib.srcv_msgrad_forward_f32(p, p, 1, 8, 9, 4, C.c_void_p(out.data_ptr()), None, 0, None) == 1
    assert lib.srcv_msgrad_forward_f32(p, p, 1, 8, 9, 4, C.c_void_p(out.data_ptr()), w, n - 256, None) != 0
    assert lib.srcv_msgrad_backward_f32(p, p, 1, 8, 9, 4, C.c_void_p(out.data_ptr()), None, w, n, None) == 1
    assert lib.srcv_si_loss_workspace_bytes(-1) == 0 and lib.srcv_si_loss_workspace_bytes(1 << 31) == 0
    m = lib.srcv_si_loss_workspace_bytes(72)
    assert lib.srcv_si_loss_forward_f32(None, p, 72, 0.85, C.c_void_p(out.data_ptr()), w, m, None) == 1
    assert lib.srcv_si_loss_forward_f32(p, p, -1, 0.85, C.c_void_p(out.data_ptr()), w, m, None) == 2
    assert lib.srcv_si_loss_forward_f32(p, p, 72, 0.85, C.c_void_p(out.data_ptr()), None, 0, None) == 1
    assert lib.srcv_si_loss_backward_f32(p, p, 72, 0.85, None, None, None, w, m, None) == 1
    for bad in (0, 5):
        with pytest.raises(ValueError, match="4"):
            L.MSGradientLoss(bad)
    with pytest.raises(ValueError):
        L.MSGradientLoss()(torch.rand(1, 1, 4, 4), torch.rand(1, 1, 4, 5))
    with pytest.raises(ValueError):
        L.MSGradientLoss()(torch.rand(1, 3, 4, 4), torch.rand(1, 3, 4, 4))
    with pytest.raises(ValueError):
        L.ScaleInvariantLoss()(torch.rand(4), torch.rand(5))


def test_launch_counts_and_determinism(emulated):
    gt, pred = _batch(9, 2, 20, 36)
    runs = []
    for _ in range(2):
        p = pred.clone().requires_grad_(True)
        c0 = _native.launch_count()
        loss = L.MSGradientLoss()(gt, p)
        c1 = _native.launch_count()
        loss.backward()
        c2 = _native.launch_count()
        assert (c1 - c0, c2 - c1) == (3, 4)                            # pyramids, partials, finalize; one per level
        runs.append((loss, p.grad))
    for x, y in zip(*runs):
        assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))
    p = pred.clone().requires_grad_(True)
    c0 = _native.launch_count()
    loss = L.MSGradientLoss(1)(gt, p)
    c1 = _native.launch_count()
    loss.backward()
    assert (c1 - c0, _native.launch_count() - c1) == (2, 1)           # no pyramid to build
    a, b = torch.randn(500, requires_grad=True), torch.randn(500, requires_grad=True)
    c0 = _native.launch_count()
    loss = L.ScaleInvariantLoss()(a, b)
    c1 = _native.launch_count()
    loss.backward()
    assert (c1 - c0, _native.launch_count() - c1) == (2, 1)


def test_modules_have_no_state():
    assert list(L.MSGradientLoss().state_dict()) == [] and list(L.MSGradientLoss().parameters()) == []
    assert list(L.ScaleInvariantLoss().state_dict()) == []
    assert L.ScaleInvariantLoss(0.5).si_lambda == 0.5 and L.MSGradientLoss(3).num_scales == 3
    assert S.MSGradientLoss is L.MSGradientLoss and S.ScaleInvariantLoss is L.ScaleInvariantLoss


def test_install_and_uninstall_on_stand_in_modules(monkeypatch):
    pkg, cv = types.ModuleType("modules"), types.ModuleType("modules.cost_volume")   # install() always patches it
    pkg.cost_volume = cv
    ref_losses = types.ModuleType("losses")
    dm = types.ModuleType("experiment_modules.depth_model")            # binds the names at import (:7)
    for n in ("MSGradientLoss", "ScaleInvariantLoss", "MVDepthLoss", "NormalsLoss"):
        setattr(ref_losses, n, type(n, (torch.nn.Module,), {}))
        setattr(dm, n, getattr(ref_losses, n))
    for name, mod in (("modules", pkg), ("modules.cost_volume", cv), ("losses", ref_losses),
                      ("experiment_modules.depth_model", dm)):
        monkeypatch.setitem(sys.modules, name, mod)
    orig = {n: getattr(ref_losses, n) for n in ("MSGradientLoss", "ScaleInvariantLoss", "MVDepthLoss", "NormalsLoss")}
    try:
        patched = S.install(depth_losses=True)
        assert "losses" in patched and "experiment_modules.depth_model" in patched
        for mod in (ref_losses, dm):
            assert mod.MSGradientLoss is L.MSGradientLoss and mod.ScaleInvariantLoss is L.ScaleInvariantLoss
            assert mod.MVDepthLoss is orig["MVDepthLoss"] and mod.NormalsLoss is orig["NormalsLoss"]
        S.uninstall()
        S.install(losses=True)                                         # the other flags keep their meaning
        assert ref_losses.MVDepthLoss is L.MVDepthLoss and ref_losses.MSGradientLoss is orig["MSGradientLoss"]
    finally:
        S.uninstall()
    for mod in (ref_losses, dm):
        assert all(getattr(mod, n) is c for n, c in orig.items())
