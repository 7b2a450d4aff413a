"""GPU: the gradient-loss kernels behind MSGradientLoss / ScaleInvariantLoss against the fp64 CPU oracle at the
training size (192x256, batch 16, options.py:70-71, :93), at 480x640 and at an odd size, with an fp16 prediction,
the terms as the training step composes them, and bitwise determinism across runs and streams."""
import pytest
import torch

from oracle import gradloss_oracle as O
from simplerecon_b200 import _native, losses as L
from simplerecon_b200.synthetic import make_normals_batch
from tests.test_emu_gradloss import check_msgrad, check_si, near_zero_footprint

pytestmark = pytest.mark.gpu


def _batch(seed, B, H, W, holes=True):
    t = make_normals_batch(seed, B, H, W, holes=holes)
    return t["depth_gt_b1hw"], t["depth_pred_b1hw"]


@pytest.mark.parametrize("seed,B,H,W", [(0, 16, 192, 256), (1, 2, 480, 640), (2, 3, 17, 23)])
def test_loss_counts_and_gradient(cuda_device, seed, B, H, W):
    gt, pred = _batch(seed, B, H, W)
    check_msgrad(gt, pred, device="cuda")
    assert _native.last_variant() == "msgrad_forward_f32"
    check_msgrad(gt, pred, num_scales=2, device="cuda")


def test_fp16_prediction(cuda_device):
    gt, pred = _batch(4, 4, 192, 256)
    loss, g = check_msgrad(gt, pred.half(), device="cuda")
    assert g.dtype == torch.float16 and loss.dtype == torch.float32


@pytest.mark.parametrize("n", [1, 7, 16 * 192 * 256 // 2])
def test_scale_invariant_loss(cuda_device, n):
    g = torch.Generator().manual_seed(n)
    gt = torch.randn(n, generator=g)
    check_si(gt, gt + 0.3 * torch.randn(n, generator=g) + 0.1, device="cuda")
    assert torch.isnan(L.ScaleInvariantLoss()(torch.empty(0, device="cuda"), torch.empty(0, device="cuda")))


def _step(gt, pred, grad_loss, si_loss):
    """depth_model.py:466-468, :487: the gradient term on the depths, the scale-invariant term on the masked logs"""
    p = pred.clone().requires_grad_(True)
    mask = torch.isfinite(gt) & (gt > 0)
    g = grad_loss(gt, p)
    si = si_loss(torch.log(gt[mask]), torch.log(p[mask]))
    (1.0 * g + si).backward()
    return g.detach(), si.detach(), p.grad


def test_training_step_composition_and_determinism(cuda_device):
    gt_c, pred_c = _batch(5, 16, 192, 256)
    gt, pred = gt_c.cuda(), pred_c.cuda()
    grad_loss, si_loss = L.MSGradientLoss(), L.ScaleInvariantLoss()
    runs = [_step(gt, pred, grad_loss, si_loss) for _ in range(2)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(_step(gt, pred, grad_loss, si_loss))
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            assert torch.equal(x, y)
    l64 = _step(gt_c.double(), pred_c.double(), O.ms_gradient_loss, O.scale_invariant_loss)
    g, si, grad = (x.cpu().double() for x in runs[0])
    assert abs(g - l64[0]) <= 2e-6 * l64[0] and abs(si - l64[1]) <= 2e-6 * l64[1]
    assert torch.isfinite(grad).all()
    bad = ((grad - l64[2]).abs() > 1e-4 * l64[2].abs().max()).sum()
    assert bad <= near_zero_footprint(gt_c.double(), pred_c.double(), 4) and bad <= 0.01 * grad.numel()


def test_cpu_tensors_are_refused():
    with pytest.raises(RuntimeError):
        L.MSGradientLoss()(torch.rand(1, 1, 8, 12), torch.rand(1, 1, 8, 12))
    with pytest.raises(RuntimeError):
        L.ScaleInvariantLoss()(torch.rand(5), torch.rand(5))
