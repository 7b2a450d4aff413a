"""GPU: the regression-loss kernels behind ``depth_regression_losses`` against the fp64 CPU oracle at the training size
(B = 16, 192x256 with scales 96x128, 48x64, 24x32), at 480x640 and at an odd size; no host synchronisation under
``torch.cuda.set_sync_debug_mode("error")`` (the reference's op sequence raises there); the whole ``compute_losses``
with every install flag against the oracle composition; bitwise determinism across runs and streams; CPU inputs."""
import sys
import types
import warnings

import pytest
import torch

import simplerecon_b200 as S
from oracle import normals_oracle
from oracle import regloss_oracle as R
from simplerecon_b200 import _native, losses as L
from simplerecon_b200.synthetic import make_training_step_batch
from tests.test_emu_regloss import check_regloss
from tests.test_regloss_oracle_vs_reference import make_inputs, step_outputs

pytestmark = pytest.mark.gpu


def _terms_inputs(seed, B, H, W):
    cur, _, out = make_training_step_batch(seed, B, H, W, views=1)
    lps = {i: out[f"log_depth_pred_s{i}_b1hw"] for i in range(4)}
    return cur["depth_b1hw"], cur["mask_b_b1hw"], lps, out["depth_pred_s0_b1hw"]


@pytest.mark.parametrize("seed,B,H,W", [(0, 16, 192, 256), (1, 2, 480, 640), (2, 3, 17, 23)])
def test_regression_terms(cuda_device, seed, B, H, W):
    gt, mask, lps, dp = _terms_inputs(seed, B, H, W)
    check_regloss(gt, mask, lps, dp, device="cuda")
    assert _native.last_variant() == "regloss_backward_f32"
    check_regloss(gt, mask, {0: lps[0], 2: lps[2]}, dp, reach=("ms_loss",), device="cuda")


@pytest.mark.parametrize("case", ["low_and_nan_preds", "zero_gt_in_mask", "empty_mask", "scale_larger_than_gt_b1_12x16"])
def test_edge_cases(cuda_device, case):
    check_regloss(*make_inputs(case), device="cuda")


def test_fp16_predictions(cuda_device):
    gt, mask, lps, dp = _terms_inputs(4, 4, 192, 256)
    out, leaves, p = check_regloss(gt, mask, {i: t.half() for i, t in lps.items()}, dp.half(), device="cuda")
    assert p.grad.dtype == torch.float16 and out["ms_loss"].dtype == torch.float32


def _cuda(d):
    return {k: v.cuda() if torch.is_tensor(v) else v for k, v in d.items()}


def test_no_host_synchronisation(cuda_device):
    gt, mask, lps, dp = (x.cuda() if torch.is_tensor(x) else _cuda(x) for x in _terms_inputs(5, 16, 192, 256))
    leaves = {i: t.clone().requires_grad_(True) for i, t in lps.items()}
    p = dp.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = L.depth_regression_losses(gt, mask, leaves, p)
        sum(out.values()).backward()
        with pytest.raises(RuntimeError):                  # the reference's boolean indexing synchronises
            R.regression_terms(gt, mask, {i: t.detach() for i, t in leaves.items()}, dp)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(out["ms_loss"]) and torch.isfinite(p.grad).all()


def _stand_in_reference(monkeypatch):
    """modules named as the reference's, holding the oracle's functions as the originals; the depth model builds its
    loss modules from the names it bound at import, as DepthModel.__init__ does (depth_model.py:139-151)"""
    from oracle import gradloss_oracle, mvdepth_oracle

    def module(fn):
        return type(fn.__name__, (torch.nn.Module,), {"forward": lambda self, *a, **k: fn(*a, **k),
                                                     "__init__": lambda self, *a, **k: torch.nn.Module.__init__(self)})

    losses = types.ModuleType("losses")
    losses.MSGradientLoss, losses.NormalsLoss = module(gradloss_oracle.ms_gradient_loss), module(normals_oracle.normals_loss)
    losses.MVDepthLoss, losses.ScaleInvariantLoss = module(mvdepth_oracle.mv_depth_loss), L.ScaleInvariantLoss
    geo = types.ModuleType("utils.geometry_utils")
    geo.NormalGenerator = S.NormalGenerator
    dm = types.ModuleType("experiment_modules.depth_model")
    for n in ("MSGradientLoss", "NormalsLoss", "MVDepthLoss", "ScaleInvariantLoss"):
        setattr(dm, n, getattr(losses, n))

    def __init__(self, height, width):
        torch.nn.Module.__init__(self)
        self.si_loss, self.grad_loss = dm.ScaleInvariantLoss(), dm.MSGradientLoss()
        self.abs_loss = torch.nn.L1Loss()
        self.normals_loss, self.mv_depth_loss = dm.NormalsLoss(), dm.MVDepthLoss(height, width)
        self.ms_loss_fn = self.abs_loss

    dm.DepthModel = type("DepthModel", (torch.nn.Module,), {"__init__": __init__,
                                                             "compute_losses": lambda self, c, s, o: R.compute_losses(c, s, o)})
    pkg, cv = types.ModuleType("modules"), types.ModuleType("modules.cost_volume")
    for name, mod in (("modules", pkg), ("modules.cost_volume", cv), ("losses", losses), ("utils.geometry_utils", geo),
                      ("experiment_modules", types.ModuleType("experiment_modules")),
                      ("experiment_modules.depth_model", dm)):
        monkeypatch.setitem(sys.modules, name, mod)
    return dm


def test_compute_losses_with_every_install_flag(cuda_device, monkeypatch):
    dm = _stand_in_reference(monkeypatch)
    B, H, W = 4, 192, 256
    cur, src, out = make_training_step_batch(6, B, H, W, views=3)
    try:
        S.install(losses=True, normals=True, depth_losses=True, regression_losses=True)
        model = dm.DepthModel(H, W)
        assert isinstance(model.grad_loss, L.MSGradientLoss) and isinstance(model.mv_depth_loss, L.MVDepthLoss)
        ng = S.NormalGenerator(H, W).cuda()
        c, s, o = _cuda(cur), _cuda(src), _cuda(out)
        c["normals_b3hw"] = ng(c["depth_b1hw"], c["invK_s0_b44"])
        ours = step_outputs(lambda *a: model.compute_losses(*a), c, s, o, ng)
        # the already-merged classes' synchronisations, reported and left as they are
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("warn")
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            step_outputs(lambda *a: model.compute_losses(*a), c, s, o, ng)
            torch.cuda.set_sync_debug_mode("default")
        print(f"\nsynchronising calls in the whole compute_losses + backward: {len(caught)}")
        for w in caught:
            print("  ", str(w.message).splitlines()[0][:160])
        # the CPU ground truth goes to the original
        ng_cpu = normals_oracle.normal_generator
        cpu = model.compute_losses(dict(cur, normals_b3hw=ng_cpu(cur["depth_b1hw"], cur["invK_s0_b44"])), src,
                                   dict(out, normals_pred_b3hw=ng_cpu(out["depth_pred_s0_b1hw"], cur["invK_s0_b44"])))
        assert list(cpu) == list(R.STEP_KEYS) and all(not v.is_cuda for v in cpu.values())
    finally:
        torch.cuda.set_sync_debug_mode("default")
        S.uninstall()
    d = lambda t: {k: v.double() if torch.is_floating_point(v) else v for k, v in t.items()}   # noqa: E731
    cur64 = d(cur)
    cur64["normals_b3hw"] = normals_oracle.normal_generator(cur64["depth_b1hw"], cur64["invK_s0_b44"])
    ref = step_outputs(lambda *a: R.compute_losses(*a), cur64, d(src), d(out), normals_oracle.normal_generator)
    assert ours["keys"].tolist() == list(range(9))
    for k in R.STEP_KEYS:
        a, b = ours[k].item(), ref[k].item()
        assert abs(a - b) <= 1e-5 * abs(b), (k, a, b)
    for i in range(4):
        g, g64 = ours[f"grad_loss_s{i}"].cpu().double(), ref[f"grad_loss_s{i}"]
        assert torch.isfinite(g).all()
        assert ((g - g64).abs() > 1e-3 * g64.abs().max()).sum() <= 0.01 * g.numel(), i


def test_determinism_across_runs_and_streams(cuda_device):
    gt, mask, lps, dp = (x.cuda() if torch.is_tensor(x) else _cuda(x) for x in _terms_inputs(7, 16, 192, 256))

    def run():
        leaves = {i: t.clone().requires_grad_(True) for i, t in lps.items()}
        p = dp.clone().requires_grad_(True)
        out = L.depth_regression_losses(gt, mask, leaves, p)
        sum(out.values()).backward()
        return [*out.values(), p.grad, *[leaves[i].grad for i in range(4)]]

    runs = [run(), run()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(run())
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            assert torch.equal(x, y)


def test_cpu_tensors_are_refused():
    gt, mask, lps, dp = _terms_inputs(8, 1, 8, 12)
    with pytest.raises(RuntimeError):
        L.depth_regression_losses(gt, mask, lps, dp)
