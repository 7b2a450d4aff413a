"""Times the depth metrics of test.py's evaluation loop (test.py:282-299) on the GPU: ground truth 480x640,
prediction 192x256, nearest resampling, valid = gt > 0.5, mult_a, at B = 1, 8 and 32.

Arms (same inputs, same stream):
  reference  the reference's op sequence as PyTorch CUDA ops: F.interpolate + gt > 0.5 + the fp32
             compute_depth_metrics_batched (oracle/metrics_oracle.py, op for op the reference's);
  fused      simplerecon_b200.depth_metrics (two launches), without and with the resampled output.
Reports the median of per-call CUDA-event times after warm-up, kernel launches per call (torch.profiler,
in a separate pass), and the algorithmic bytes per call (4 H W gt + 4 Hp Wp prediction, + 4 H W when the
resampled map is written) as a share of the H100 SXM data sheet's 3.35 TB/s.  Prints the card's name
and power limit with the numbers, one JSON line per (arm, B).

    python scripts/bench_metrics.py [--iters 200] [--warmup 20]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import simplerecon_b200 as S  # noqa: E402
from oracle import metrics_oracle as M  # noqa: E402

H, W, HP, WP = 480, 640, 192, 256
PEAK_BPS = 3.35e12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().splitlines() or ["? , ? , ?"])[0].split(", ")[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def reference_arm(gt, pred):
    up = F.interpolate(pred, size=gt.shape[-2:], mode="nearest")
    valid = gt > 0.5
    return M.compute_depth_metrics_batched(gt.flatten(1).float(), up.flatten(1).float(), valid.flatten(1), mult_a=True)


def fused_arm(gt, pred):
    return S.depth_metrics(gt, pred, min_valid_depth=0.5, mult_a=True)


def fused_up_arm(gt, pred):
    return S.depth_metrics(gt, pred, min_valid_depth=0.5, mult_a=True, return_upsampled=True)


def time_ms(fn, args, iters, warmup):
    for _ in range(warmup):
        fn(*args)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn(*args)
        b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ev)


def launches_per_call(fn, args, calls=5):
    from torch.profiler import ProfilerActivity, profile
    fn(*args)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn(*args)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and
               "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
    return len(kernels) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batches", default="1,8,32")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_metrics.py measures on the GPU; there is no CPU timing"
    info = card()
    for B in map(int, a.batches.split(",")):
        g = torch.Generator(device="cuda").manual_seed(B)
        gt = torch.rand(B, 1, H, W, device="cuda", generator=g) * 6
        pred = torch.rand(B, 1, HP, WP, device="cuda", generator=g) * 6 + 0.05
        m, c = fused_arm(gt, pred)                        # same numbers as the reference arm
        r = reference_arm(gt, pred)
        a_err = max((m[:, 5 + i] - r[k]).abs().max().item() for i, k in enumerate(M.KEYS[5:]))
        c_err = max(((m[:, i] - r[k]).abs() / r[k].abs()).max().item() for i, k in enumerate(M.KEYS[:5]))
        for arm, fn, out_bytes in (("reference", reference_arm, 0), ("fused", fused_arm, 0),
                                   ("fused+upsampled", fused_up_arm, 4 * H * W)):
            ms = time_ms(fn, (gt, pred), a.iters, a.warmup)
            nbytes = B * (4 * H * W + 4 * HP * WP + out_bytes)
            rec = {"arm": arm, "B": B, "median_ms": round(ms, 4), "launches_per_call": launches_per_call(fn, (gt, pred)),
                   "algorithmic_MB": round(nbytes / 1e6, 2), "GBps": round(nbytes / ms / 1e6, 1),
                   "share_of_3.35TBps": round(nbytes / (ms * 1e-3) / PEAK_BPS, 3),
                   "a_metrics_max_abs_diff_vs_reference": a_err, "continuous_max_rel_diff_vs_reference": c_err, **info}
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
