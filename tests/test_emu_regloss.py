"""CPU: the regression-loss kernels (csrc/srcv_regloss.cuh) compiled for the host (tests/emu) behind
``depth_regression_losses``, against the fp64 oracle (oracle/regloss_oracle.py): the five losses, the mask counts n and
m, the gradients to every scale and to ``depth_pred``, fp16 inputs, outputs reached in part, launch counts, bitwise
determinism, the C ABI's argument checks, the drop-in ``compute_losses``, its fallback predicate, and
install()/uninstall()."""
import contextlib
import ctypes as C
import sys
import types

import pytest
import torch

import simplerecon_b200 as S
from oracle import gradloss_oracle, mvdepth_oracle, normals_oracle
from oracle import regloss_oracle as R
from simplerecon_b200 import _native, losses as L
from simplerecon_b200.synthetic import make_training_step_batch
from tests import emu
from tests.test_regloss_oracle_vs_reference import CASES, make_inputs


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


def counts(gt, mask, lps, dp, si_lambda=0.85):
    """(n, m) as the forward leaves them in the workspace"""
    dev = gt.device
    f32 = lambda t: t.float().contiguous()   # noqa: E731
    keep = [f32(gt), mask.contiguous().view(torch.uint8), f32(dp)] + [f32(lps[i]) if i in lps else None for i in range(4)]
    args, ws = L._regloss_call(keep[0], keep[1], keep[2], keep[3:], si_lambda)
    out = torch.empty(5, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _native.check(_native.load().srcv_regloss_forward_f32(C.byref(args), C.c_void_p(out.data_ptr()),
                                                             C.c_void_p(ws.data_ptr()), ws.numel(), L._stream(dev)))
    return tuple(ws[:16].cpu().view(torch.int64).tolist())


def near_zero(gt, mask, lps, dp):
    """How many gradient elements a sign flip of a near-zero difference can move: the masked pixels where a term's
    fp64 difference is within fp32 rounding of zero (each flips one element of one gradient)."""
    gt, dp = gt.double(), dp.double()
    lg = torch.log(gt)
    H, W = gt.shape[-2:]
    total = 0
    for t in lps.values():
        r = torch.nn.functional.interpolate(t.double(), size=(H, W), mode="nearest")
        total += int((mask & ((lg - r).abs() <= 1e-6 * max(1.0, lg[mask].abs().max().item() if mask.any() else 1.0))).sum())
    total += int((mask & ((gt - dp).abs() <= 1e-6 * gt[mask].abs().max().clamp_min(1.0))).sum()) if mask.any() else 0
    total += int((mask & ((1 / gt - 1 / dp).abs() <= 1e-5)).sum())
    return total


def check_regloss(gt, mask, lps, dp, reach=R.KEYS, si_lambda=0.85, device="cpu"):
    """the fused call against the fp64 oracle; ``reach`` lists the outputs the backward starts from (sum of them):
      - n and m exact (from the workspace);
      - every loss within 2e-6 relative of the fp64 oracle, or within twice the fp32 oracle's own error, NaN exactly
        where the oracle's is;
      - each gradient NaN exactly where the oracle's is, elsewhere within 1e-4 of its max |g64| (plus the input
        dtype's rounding), except at most `near_zero` elements."""
    leaves = {i: t.to(device).clone().requires_grad_(True) for i, t in lps.items()}
    p = dp.to(device).clone().requires_grad_(True)
    out = L.depth_regression_losses(gt.to(device), mask.to(device), leaves, p, si_lambda)
    assert list(out) == list(R.KEYS)
    assert all(v.dtype == torch.float32 and v.shape == () and v.device == p.device for v in out.values())
    assert counts(gt.to(device), mask.to(device), {i: t.to(device) for i, t in lps.items()}, p.detach()) == \
        R.masks(gt, mask, dp)
    if reach:
        sum(out[k] for k in reach).backward()
    l64_leaves = {i: t.double().clone().requires_grad_(True) for i, t in lps.items()}
    p64 = dp.double().clone().requires_grad_(True)
    l64 = R.regression_terms(gt.double(), mask, l64_leaves, p64, si_lambda)
    l32 = R.regression_terms(gt.float(), mask, {i: t.float() for i, t in lps.items()}, dp.float(), si_lambda)
    if reach:
        sum(l64[k] for k in reach).backward()
    for k in R.KEYS:
        a, b, c = out[k].item(), l64[k].item(), l32[k].item()
        if b != b:
            assert a != a, k
        elif abs(b) == float("inf"):                                    # log(0) inside the mask
            assert a == b, k
        else:
            assert abs(a - b) <= max(2e-6 * abs(b), 2 * abs(c - b) + 1e-6 * abs(b)), (k, a, b, c)
    bound = near_zero(gt, mask, lps, dp)
    pairs = [(leaves[i], l64_leaves[i]) for i in lps] + [(p, p64)]
    for x, x64 in pairs:
        g = x.grad
        if not reach:
            assert g is None
            continue
        g64 = x64.grad if x64.grad is not None else torch.zeros_like(x64)
        assert g is not None and g.dtype == x.dtype and g.shape == x.shape
        g = g.cpu().double()
        assert torch.equal(g.isnan(), g64.isnan())
        fin = ~g64.isnan()
        scale = g64[fin].abs().max().item() if fin.any() else 0.0
        # a half / bfloat16 gradient was rounded to that dtype: its relative step, and its subnormal spacing (a mean
        # over 10^5 pixels puts the gradient below fp16's smallest normal)
        fi = torch.finfo(x.dtype)
        half, spacing = (fi.eps, fi.smallest_normal * fi.eps) if x.dtype != torch.float32 else (0.0, 0.0)
        bad = int(((g - g64).abs()[fin] > (1e-4 + half) * scale + spacing + 1e-30).sum())
        assert bad <= bound, (bad, bound, scale)
    return out, leaves, p


@pytest.mark.parametrize("case", list(CASES))
def test_golden_cases(emulated, case):
    gt, mask, lps, dp = make_inputs(case)
    check_regloss(gt, mask, lps, dp)
    check_regloss(gt, mask, lps, dp, reach=("ms_loss", "abs_loss", "inv_abs_loss", "log_l1_loss"))


@pytest.mark.parametrize("seed,B,H,W,sizes", [
    (0, 16, 24, 32, [(12, 16), (6, 8), (3, 4)]),
    (1, 3, 13, 29, [(7, 15), (4, 8), (2, 4)]),
    (2, 1, 31, 9, [(31, 9), (10, 3), (1, 1)]),          # a same-size scale and a 1x1 one
    (3, 2, 10, 14, [(21, 29), None, (3, 40)]),          # upsampled scales: coarse pixels with empty preimages
])
def test_ragged_sizes_and_batches(emulated, seed, B, H, W, sizes):
    cur, _, out = make_training_step_batch(seed, B, H, W, views=1)
    g = torch.Generator().manual_seed(seed)
    s0 = out["log_depth_pred_s0_b1hw"]
    lps = {0: s0}
    for i, hw in enumerate(sizes, start=1):
        if hw is not None:
            lps[i] = (torch.nn.functional.adaptive_avg_pool2d(s0, hw) if hw[0] <= H and hw[1] <= W
                      else torch.nn.functional.interpolate(s0, size=hw, mode="bilinear")) + \
                0.03 * torch.randn(B, 1, *hw, generator=g)
    check_regloss(cur["depth_b1hw"], cur["mask_b_b1hw"], lps, out["depth_pred_s0_b1hw"])


def test_outputs_reached_in_part(emulated):
    gt, mask, lps, dp = make_inputs("b2_24x32")
    for reach in (("ms_loss",), ("si_loss",), ("abs_loss", "inv_abs_loss"), ("log_l1_loss", "si_loss"), ()):
        check_regloss(gt, mask, lps, dp, reach=reach)
    # the NaN si_loss of a NaN prediction poisons only what reaches it
    gt, mask, lps, dp = make_inputs("low_and_nan_preds")
    _, leaves, p = check_regloss(gt, mask, lps, dp, reach=("ms_loss", "abs_loss"))
    assert torch.isfinite(leaves[0].grad).all() and torch.isfinite(p.grad).all()


def test_half_inputs(emulated):
    gt, mask, lps, dp = make_inputs("odd_b1_17x23")
    _, leaves, p = check_regloss(gt, mask, {i: t.half() for i, t in lps.items()}, dp.half())
    assert p.grad.dtype == torch.float16 and leaves[2].grad.dtype == torch.float16
    _, leaves, p = check_regloss(gt, mask, {i: t.bfloat16() for i, t in lps.items()}, dp)
    assert p.grad.dtype == torch.float32 and leaves[0].grad.dtype == torch.bfloat16


def test_launch_counts_and_determinism(emulated):
    gt, mask, lps, dp = make_inputs("b2_24x32")
    runs = []
    for _ in range(2):
        leaves = {i: t.clone().requires_grad_(True) for i, t in lps.items()}
        p = dp.clone().requires_grad_(True)
        c0 = _native.launch_count()
        out = L.depth_regression_losses(gt, mask, leaves, p)
        c1 = _native.launch_count()
        sum(out.values()).backward()
        c2 = _native.launch_count()
        assert (c1 - c0, c2 - c1) == (2, 1)
        runs.append([*out.values(), p.grad, *[leaves[i].grad for i in sorted(leaves)]])
    for x, y in zip(*runs):
        assert torch.equal(x, y)


def test_argument_checks(emulated):
    lib = emulated
    B, H, W = 1, 8, 9
    gt, dp = torch.rand(B, 1, H, W) + 0.5, torch.rand(B, 1, H, W) + 0.5
    mask = torch.ones(B, 1, H, W, dtype=torch.uint8)
    lp = [torch.rand(B, 1, H, W), torch.rand(B, 1, 4, 5)]
    out = torch.empty(5)

    def args(log0=True, h0=H, w0=W, h1=4, w1=5, B_=B, H_=H, W_=W):
        return _native.RegLossArgs(gt.data_ptr(), mask.data_ptr(), dp.data_ptr(),
                                   (C.c_void_p * 4)(lp[0].data_ptr() if log0 else None, lp[1].data_ptr(), None, None),
                                   (C.c_int32 * 4)(h0, h1, 0, 0), (C.c_int32 * 4)(w0, w1, 0, 0), B_, H_, W_, 0.85)

    a = args()
    n = lib.srcv_regloss_workspace_bytes(C.byref(a))
    ws = torch.empty(n, dtype=torch.uint8)
    w = C.c_void_p(ws.data_ptr())
    o = C.c_void_p(out.data_ptr())
    assert lib.srcv_regloss_forward_f32(C.byref(a), o, w, n, None) == 0
    assert lib.srcv_regloss_forward_f32(C.byref(args(log0=False)), o, w, n, None) == 1      # scale 0 is required
    assert lib.srcv_regloss_workspace_bytes(C.byref(args(log0=False))) == 0
    for bad in (args(h0=H - 1), args(w0=W + 1), args(h1=0), args(w1=0), args(B_=70000), args(B_=0), args(H_=0),
                args(h0=1 << 14, w0=1 << 14, B_=4, H_=1 << 14, W_=1 << 14)):
        assert lib.srcv_regloss_workspace_bytes(C.byref(bad)) == 0
        assert lib.srcv_regloss_forward_f32(C.byref(bad), o, w, n, None) == 2
    assert lib.srcv_regloss_forward_f32(None, o, w, n, None) == 1
    assert lib.srcv_regloss_forward_f32(C.byref(a), None, w, n, None) == 1
    assert lib.srcv_regloss_forward_f32(C.byref(a), o, None, 0, None) == 1
    assert lib.srcv_regloss_forward_f32(C.byref(a), o, w, n - 256, None) == 3
    g5, g4 = (C.c_void_p * 5)(), (C.c_void_p * 4)()
    assert lib.srcv_regloss_backward_f32(C.byref(a), g5, g4, None, w, n, None) == 0       # nothing wanted
    assert lib.srcv_regloss_backward_f32(C.byref(a), None, g4, None, w, n, None) == 1
    with pytest.raises(ValueError, match="scale 0"):
        L.depth_regression_losses(gt, mask.bool(), {1: lp[1]}, dp)
    with pytest.raises(ValueError):
        L.depth_regression_losses(gt, mask.bool(), {0: lp[1]}, dp)                      # scale 0 of another size
    with pytest.raises(ValueError):
        L.depth_regression_losses(gt, mask, {0: lp[0]}, dp)                             # not a bool mask
    with pytest.raises(ValueError):
        L.depth_regression_losses(gt, mask.bool(), {0: lp[0], 4: lp[1]}, dp)
    with pytest.raises(ValueError):
        L.depth_regression_losses(gt, mask.bool(), {0: lp[0], 1: torch.rand(B, 1, 0, 5)}, dp)


class _FakeCuda(torch.Tensor):
    @property
    def is_cuda(self):
        return True


def test_fallback_predicate():
    gt = torch.zeros(1, 1, 2, 2)
    l1 = torch.nn.L1Loss()
    model = lambda ms, ab: types.SimpleNamespace(ms_loss_fn=ms, abs_loss=ab)   # noqa: E731
    assert L.uses_fused_regression_losses(model(l1, l1), gt.as_subclass(_FakeCuda))
    assert not L.uses_fused_regression_losses(model(l1, l1), gt)                              # CPU ground truth
    assert not L.uses_fused_regression_losses(model(torch.nn.L1Loss(), l1), gt.as_subclass(_FakeCuda))
    s = torch.nn.L1Loss(reduction="sum")
    assert not L.uses_fused_regression_losses(model(s, s), gt.as_subclass(_FakeCuda))
    mse = torch.nn.MSELoss()
    assert not L.uses_fused_regression_losses(model(mse, mse), gt.as_subclass(_FakeCuda))


def _oracle_model(si_lambda=0.85):
    l1 = torch.nn.L1Loss()
    return types.SimpleNamespace(si_loss=types.SimpleNamespace(si_lambda=si_lambda), abs_loss=l1, ms_loss_fn=l1,
                                 grad_loss=gradloss_oracle.ms_gradient_loss, normals_loss=normals_oracle.normals_loss,
                                 mv_depth_loss=mvdepth_oracle.mv_depth_loss)


def test_compute_losses_on_the_kernels(emulated, monkeypatch):
    """the drop-in compute_losses with the emulated kernels for the regression terms and the oracles for the other
    three, against the oracle composition in fp64: keys, order, values and the gradient of `loss` to the scales"""
    monkeypatch.setattr(L, "uses_fused_regression_losses", lambda model, gt: True)
    from tests.test_regloss_oracle_vs_reference import step_outputs
    cur, src, out = make_training_step_batch(3, 2, 48, 64, views=2)
    cur["normals_b3hw"] = normals_oracle.normal_generator(cur["depth_b1hw"], cur["invK_s0_b44"])
    ours = step_outputs(lambda c, s, o: L.compute_losses(_oracle_model(), c, s, o), cur, src, out,
                        normals_oracle.normal_generator)
    d = lambda t: {k: v.double() if torch.is_floating_point(v) else v for k, v in t.items()}   # noqa: E731
    ref = step_outputs(lambda c, s, o: R.compute_losses(c, s, o), d(cur), d(src), d(out),
                       normals_oracle.normal_generator)
    assert ours["keys"].tolist() == list(range(9))
    for k in R.STEP_KEYS:
        assert abs(ours[k].item() - ref[k].item()) <= 1e-5 * abs(ref[k].item()), k
    for i in range(4):
        g, g64 = ours[f"grad_loss_s{i}"].double(), ref[f"grad_loss_s{i}"]
        assert ((g - g64).abs() > 1e-3 * g64.abs().max()).sum() <= 0.01 * g.numel(), i
    with pytest.raises(Exception, match="Could not find a valid scale"):
        L.compute_losses(_oracle_model(), cur, src, {"depth_pred_s0_b1hw": out["depth_pred_s0_b1hw"]})


def test_install_and_uninstall_on_stand_in_modules(monkeypatch):
    pkg, cv = types.ModuleType("modules"), types.ModuleType("modules.cost_volume")   # install() always patches it
    pkg.cost_volume = cv
    em, dm = types.ModuleType("experiment_modules"), types.ModuleType("experiment_modules.depth_model")
    em.depth_model = dm
    sentinel = {"original": True}

    def original(self, cur_data, src_data, outputs):
        return sentinel

    dm.DepthModel = type("DepthModel", (torch.nn.Module,), {"compute_losses": original})
    ref_losses = types.ModuleType("losses")
    ref_losses.MVDepthLoss = dm.MVDepthLoss = type("MVDepthLoss", (torch.nn.Module,), {})
    for name, mod in (("modules", pkg), ("modules.cost_volume", cv), ("experiment_modules", em),
                      ("experiment_modules.depth_model", dm), ("losses", ref_losses)):
        monkeypatch.setitem(sys.modules, name, mod)
    try:
        patched = S.install(regression_losses=True)
        assert "experiment_modules.depth_model" in patched
        assert dm.DepthModel.compute_losses is L.compute_losses
        assert dm.MVDepthLoss is ref_losses.MVDepthLoss                # the other flags keep their meaning
        model = _oracle_model()
        cur, src, out = make_training_step_batch(0, 1, 8, 12, views=1)
        assert dm.DepthModel.compute_losses(model, cur, src, out) is sentinel    # CPU ground truth -> the original
        S.uninstall()
        assert dm.DepthModel.compute_losses is original
        S.install(losses=True, regression_losses=True)
        assert dm.MVDepthLoss is L.MVDepthLoss and dm.DepthModel.compute_losses is L.compute_losses
    finally:
        S.uninstall()
    assert dm.DepthModel.compute_losses is original and dm.MVDepthLoss is ref_losses.MVDepthLoss
    with pytest.raises(RuntimeError, match="not been replaced"):
        L.compute_losses(_oracle_model(), cur, src, out)
