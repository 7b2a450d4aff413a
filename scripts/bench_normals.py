"""Times the normals work of one training step (experiment_modules/depth_model.py:526-530, :475): NormalGenerator
on the ground truth without grad, NormalGenerator on the prediction, NormalsLoss, and the backward to the predicted
depth — the kernels (csrc/srcv_normals.cuh) against the oracle's fp32 op sequence (the reference's ops) run as
PyTorch CUDA ops on the same GPU.  CUDA events, warm-up, rotating input sets, the two arms' outputs compared;
launches per step (srcv_launch_count for ours, torch.profiler for the port), algorithmic bytes and their share of
3.35 TB/s, and the card name and power limit read in the same run.  One JSON line per batch size.

    python scripts/bench_normals.py [--batches 16 1] [--height 192] [--width 256] [--steps 50]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import simplerecon_b200 as S  # noqa: E402
from oracle import normals_oracle as O  # noqa: E402  (the comparison arm: the reference's op sequence)
from simplerecon_b200 import _native  # noqa: E402
from simplerecon_b200.synthetic import make_normals_batch  # noqa: E402

PEAK_BPS = 3.35e12
# per pixel: NG forward x2 (4 read + 12 write each), loss forward (24), loss backward (24 + 12 write),
# NG backward (a: 4 + 12 read, 24 write; b: 24 read, 4 write)
BYTES_PER_PIXEL = 2 * 16 + 24 + 36 + 40 + 28


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().splitlines() or ["? , ? , ?"])[0].split(", ")[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def step_ours(ng, crit):
    def run(gt, pred, invK):
        p = pred.clone().requires_grad_(True)
        with torch.no_grad():
            n_gt = ng(gt, invK)
        loss = crit(n_gt, ng(p, invK))
        loss.backward()
        return loss.detach(), p.grad
    return run


def step_port(gt, pred, invK):
    p = pred.clone().requires_grad_(True)
    with torch.no_grad():
        n_gt = O.normal_generator(gt, invK)
    loss = O.normals_loss(n_gt, O.normal_generator(p, invK))
    loss.backward()
    return loss.detach(), p.grad


def timed(fn, sets, steps, warmup):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for it in range(warmup + steps):
        t = sets[it % len(sets)]
        torch.cuda.synchronize()
        ev[0].record()
        out = fn(*t)
        ev[1].record()
        torch.cuda.synchronize()
        if it >= warmup:
            times.append(ev[0].elapsed_time(ev[1]))
    times.sort()
    return times[len(times) // 2], times[0], out


def port_launches(sets):
    from torch.profiler import ProfilerActivity, profile
    step_port(*sets[0])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step_port(*sets[0])
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 1])
    ap.add_argument("--height", type=int, default=192)
    ap.add_argument("--width", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    info = card()
    ng, crit = S.NormalGenerator(a.height, a.width).cuda(), S.NormalsLoss()
    ours = step_ours(ng, crit)
    for B in a.batches:
        sets = []
        for i in range(3):
            t = make_normals_batch(70 + i, B, a.height, a.width)
            sets.append((t["depth_gt_b1hw"].cuda(), t["depth_pred_b1hw"].cuda(), t["invK_b44"].cuda()))
        ms, ms_min, (l_ours, g_ours) = timed(ours, sets, a.steps, a.warmup)
        c0 = _native.launch_count()
        ours(*sets[0])
        torch.cuda.synchronize()
        launches = _native.launch_count() - c0
        ms_port, ms_port_min, _ = timed(step_port, sets, max(5, a.steps // 2), max(3, a.warmup // 2))
        l_port, g_port = step_port(*sets[(a.warmup + a.steps - 1) % len(sets)])
        alg = B * a.height * a.width * BYTES_PER_PIXEL
        print(json.dumps({
            "what": "normals step: NG(gt) no-grad + NG(pred) + NormalsLoss + backward", "batch": B,
            "hw": [a.height, a.width], **info,
            "ours_ms_median": round(ms, 4), "ours_ms_min": round(ms_min, 4),
            "port_ms_median": round(ms_port, 4), "port_ms_min": round(ms_port_min, 4),
            "speedup_median": round(ms_port / ms, 1),
            "launches_ours": launches, "launches_port": port_launches(sets),
            "loss_ours": l_ours.item(), "loss_port": l_port.item(),
            "max_abs_grad_diff": (g_ours - g_port).abs().max().item(), "max_abs_grad": g_port.abs().max().item(),
            "algorithmic_bytes": alg, "share_of_3.35TBps_at_ours_median": round(alg / (ms * 1e-3) / PEAK_BPS, 4),
        }))


if __name__ == "__main__":
    main()
