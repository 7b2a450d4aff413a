"""Times the regression terms of one training step (experiment_modules/depth_model.py:447-474) and the whole
``compute_losses`` (:409-500), each with its backward, against the reference's op sequence on the same GPU.

  terms: ``depth_regression_losses`` (csrc/srcv_regloss.cuh) against the oracle's fp32 restatement of the reference's
         ops (``F.interpolate``, boolean indexing, ``nn.L1Loss``, the scale-invariant arithmetic), both with the
         backward from ``ms_loss``, the one term of the five that the training loss contains.
  step : depth_pred = exp(s0), its normals, ``compute_losses`` and ``loss.backward()``, with the kernel-backed classes
         that ``install(losses=True, normals=True, depth_losses=True, regression_losses=True)`` puts in place, against
         the oracles' restatement of the reference's classes and ``compute_losses``.

The arms alternate step by step in one process.  CUDA events, warm-up, three rotating input sets, the arms' outputs
compared; launches and device-to-host copies per step from torch.profiler in a separate pass (a host synchronisation
of boolean indexing shows up as one such copy; the op sequence runs with PyTorch's defaults); the card name, power
limit and maximum SM clock read in the same run.  One JSON line per workload and batch size.  Needs a GPU: there is no
fallback.

    python scripts/bench_regloss.py [--batches 16 1] [--height 192] [--width 256] [--steps 50] [--warmup 10]
"""
import argparse
import json
import sys
import types
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import simplerecon_b200 as S  # noqa: E402
from oracle import normals_oracle  # noqa: E402  (the reference's op sequences)
from oracle import regloss_oracle as R  # noqa: E402
from scripts.bench_gradloss import card, timed, trace  # noqa: E402
from simplerecon_b200 import _native, losses as L  # noqa: E402
from simplerecon_b200.synthetic import make_training_step_batch  # noqa: E402


def terms_arm(fn):
    def run(cur, src, out):
        leaves = {i: out[f"log_depth_pred_s{i}_b1hw"].detach().requires_grad_(True) for i in range(4)}
        t = fn(cur["depth_b1hw"], cur["mask_b_b1hw"], leaves, out["depth_pred_s0_b1hw"])
        t["ms_loss"].backward()
        return torch.stack([t[k].detach() for k in R.KEYS]), leaves[1].grad
    return run


def step_arm(model, normal_generator):
    def run(cur, src, out):
        leaves = {i: out[f"log_depth_pred_s{i}_b1hw"].detach().requires_grad_(True) for i in range(4)}
        o = {f"log_depth_pred_s{i}_b1hw": t for i, t in leaves.items()}
        o["depth_pred_s0_b1hw"] = torch.exp(leaves[0])
        o["normals_pred_b3hw"] = normal_generator(o["depth_pred_s0_b1hw"], cur["invK_s0_b44"])
        losses = model(cur, src, o)
        losses["loss"].backward()
        return torch.stack([losses[k].detach() for k in R.STEP_KEYS]), leaves[1].grad
    return run


def report(what, B, hw, info, ours, port, sets, steps, warmup):
    (ms, ms_min, (v_ours, g_ours)), (ms_port, ms_port_min, (v_port, g_port)) = timed([ours, port], sets, steps, warmup)
    c0 = _native.launch_count()
    ours(*sets[0])
    torch.cuda.synchronize()
    counted = _native.launch_count() - c0
    k_ours, k_own, d2h_ours = trace(ours, sets[0])
    k_port, _, d2h_port = trace(port, sets[0])
    print(json.dumps({
        "what": what, "batch": B, "hw": hw, **info,
        "ours_ms_median": round(ms, 4), "ours_ms_min": round(ms_min, 4),
        "port_ms_median": round(ms_port, 4), "port_ms_min": round(ms_port_min, 4),
        "speedup_median": round(ms_port / ms, 1),
        "launches_ours": k_ours, "of_which_this_library": k_own, "counted_by_the_library": counted,
        "launches_port": k_port, "d2h_copies_ours": d2h_ours, "d2h_copies_port": d2h_port,
        "values_ours": [round(x, 6) for x in v_ours.tolist()], "values_port": [round(x, 6) for x in v_port.tolist()],
        "max_abs_grad_diff_s1": (g_ours - g_port).abs().max().item(), "max_abs_grad_s1": g_port.abs().max().item(),
    }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 1])
    ap.add_argument("--height", type=int, default=192)
    ap.add_argument("--width", type=int, default=256)
    ap.add_argument("--views", type=int, default=7)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_regloss.py needs a CUDA device")
    info = card()
    H, W = a.height, a.width
    l1 = torch.nn.L1Loss()
    ours_model = types.SimpleNamespace(si_loss=S.ScaleInvariantLoss(), grad_loss=S.MSGradientLoss(), abs_loss=l1,
                                       ms_loss_fn=l1, normals_loss=S.NormalsLoss(), mv_depth_loss=S.MVDepthLoss(H, W))
    ng = S.NormalGenerator(H, W).cuda()
    terms_ours = terms_arm(L.depth_regression_losses)
    terms_port = terms_arm(R.regression_terms)
    step_ours = step_arm(lambda c, s, o: L.compute_losses(ours_model, c, s, o), ng)
    step_port = step_arm(lambda c, s, o: R.compute_losses(c, s, o, ours_model.si_loss.si_lambda),
                         normals_oracle.normal_generator)
    for B in a.batches:
        sets = []
        for i in range(3):
            cur, src, out = make_training_step_batch(80 + i, B, H, W, views=a.views)
            cur, src, out = ({k: v.cuda() for k, v in d.items()} for d in (cur, src, out))
            with torch.no_grad():
                cur["normals_b3hw"] = ng(cur["depth_b1hw"], cur["invK_s0_b44"])
            sets.append((cur, src, out))
        report("regression terms (5) + backward from ms_loss", B, [H, W], info, terms_ours, terms_port, sets,
               a.steps, a.warmup)
        report("exp, normals, compute_losses (9) + backward from loss, every install flag", B, [H, W], info,
               step_ours, step_port, sets, a.steps, a.warmup)


if __name__ == "__main__":
    main()
