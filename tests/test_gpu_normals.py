"""GPU: the normals kernels behind NormalGenerator / NormalsLoss against the fp64 CPU oracle at the training
resolution (192x256, batch 16, options.py:70-71, :93) and at 480x640, with fp16 depth, the training step's
composition, and bitwise determinism across runs and streams."""
import pytest
import torch

from oracle import normals_oracle as O
from simplerecon_b200 import _native, normals as NM
from simplerecon_b200.synthetic import make_normals_batch
from tests.test_emu_normals import check_depth_gradient, check_loss, check_normals

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed,B,H,W", [(0, 16, 192, 256), (1, 2, 480, 640), (2, 3, 17, 23)])
def test_normals_loss_and_gradients(cuda_device, seed, B, H, W):
    t = make_normals_batch(seed, B, H, W)
    gt, pred, invK = t["depth_gt_b1hw"], t["depth_pred_b1hw"], t["invK_b44"]
    n_gt = check_normals(gt, invK, device="cuda")
    n_pred = check_normals(pred, invK, device="cuda")
    assert _native.last_variant() == "normals_forward_f32"
    check_depth_gradient(pred, invK, device="cuda", seed=seed)
    check_depth_gradient(torch.where(torch.isnan(gt), gt, pred), invK, device="cuda", seed=seed + 1)
    check_loss(n_gt, n_pred, device="cuda")


@pytest.mark.parametrize("k,sigma", [(3, 1.0), (7, 3.0), (15, 5.0)])
def test_other_kernel_sizes(cuda_device, k, sigma):
    t = make_normals_batch(3, 2, 40, 56)
    check_normals(t["depth_gt_b1hw"], t["invK_b44"], k, sigma, device="cuda")
    check_depth_gradient(t["depth_pred_b1hw"], t["invK_b44"], k, sigma, device="cuda")


def test_fp16_depth(cuda_device):
    t = make_normals_batch(4, 4, 192, 256, holes=False)
    d = t["depth_pred_b1hw"].half().cuda().requires_grad_(True)
    invK = t["invK_b44"].cuda()
    n = NM.NormalGenerator(192, 256).cuda()(d, invK)
    assert n.dtype == torch.float16
    n64 = O.normal_generator(d.detach().cpu().double(), invK.cpu().double())
    assert (n.cpu().double() - n64).abs().max() <= 2e-3
    n.float().sum().backward()
    assert d.grad.dtype == torch.float16 and torch.isfinite(d.grad).all()


def _step(gt, pred, invK, ng, crit):
    p = pred.clone().requires_grad_(True)
    n_gt = ng(gt, invK)
    n_p = ng(p, invK)
    loss = crit(n_gt, n_p)
    loss.backward()
    return n_gt, n_p, loss.detach(), p.grad


def test_training_step_composition_and_determinism(cuda_device):
    """NormalsLoss(NG(gt with NaN holes), NG(pred)) and d loss / d pred against the fp64 oracle; two runs and a
    run on a side stream give the same bits"""
    t = make_normals_batch(5, 16, 192, 256)
    gt, pred, invK = t["depth_gt_b1hw"].cuda(), t["depth_pred_b1hw"].cuda(), t["invK_b44"].cuda()
    ng, crit = NM.NormalGenerator(192, 256).cuda(), NM.NormalsLoss()
    runs = [_step(gt, pred, invK, ng, crit) for _ in range(2)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(_step(gt, pred, invK, ng, crit))
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))
    p64 = t["depth_pred_b1hw"].double().requires_grad_(True)
    i64 = t["invK_b44"].double()
    l64 = O.normals_loss(O.normal_generator(t["depth_gt_b1hw"].double(), i64), O.normal_generator(p64, i64))
    l64.backward()
    loss, g = runs[0][2].item(), runs[0][3].cpu().double()
    assert abs(loss - l64.item()) <= 2e-5 * l64.item()
    assert torch.isfinite(g).all() and (g - p64.grad).abs().max() <= 1e-4 * p64.grad.abs().max()


def test_cpu_tensors_are_refused():
    with pytest.raises(RuntimeError):
        NM.NormalGenerator(8, 12)(torch.rand(1, 1, 8, 12), torch.eye(4)[None])
    with pytest.raises(RuntimeError):
        NM.NormalsLoss()(torch.rand(1, 3, 8, 12), torch.rand(1, 3, 8, 12))
