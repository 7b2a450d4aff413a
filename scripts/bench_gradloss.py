"""Times the gradient term of one training step (experiment_modules/depth_model.py:466, :487): MSGradientLoss(gt,
pred) and the backward to the predicted depth — the kernels (csrc/srcv_gradloss.cuh) against the oracle's fp32 op
sequence (the reference's ops) run as PyTorch CUDA ops on the same GPU — and, separately, ScaleInvariantLoss on
B H W / 2 elements with its backward (:468).  The arms alternate in one process.  CUDA events, warm-up, rotating
input sets, the two arms' outputs compared; launches per step (torch.profiler's CUDA kernel events, in a separate
pass, for both arms; srcv_launch_count beside it for ours), device-to-host copies in the same trace (a host
synchronisation of the op sequence shows up as one; the op sequence runs with PyTorch's defaults, under which cuDNN
convolutions may use TF32), and the card name, power limit and maximum SM clock read in
the same run.  One JSON line per batch size and loss.  Needs a GPU: there is no fallback.

    python scripts/bench_gradloss.py [--batches 16 1] [--height 192] [--width 256] [--steps 50]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import simplerecon_b200 as S  # noqa: E402
from oracle import gradloss_oracle as O  # noqa: E402  (the comparison arm: the reference's op sequence)
from simplerecon_b200 import _native  # noqa: E402
from simplerecon_b200.synthetic import make_normals_batch  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().splitlines() or ["? , ? , ?"])[0].split(", ")[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def step(loss_fn, grads_of=(1,)):
    """loss_fn(a, b) and its backward to the inputs listed in `grads_of`"""
    def run(a, b):
        t = [a, b]
        for i in grads_of:
            t[i] = t[i].detach().requires_grad_(True)
        loss = loss_fn(*t)
        loss.backward()
        return loss.detach(), t[grads_of[-1]].grad
    return run


def timed(arms, sets, steps, warmup):
    """the arms alternate step by step; per arm (median ms, min ms, last output)"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times, out = [[] for _ in arms], [None for _ in arms]
    for it in range(warmup + steps):
        t = sets[it % len(sets)]
        for k, fn in enumerate(arms):
            torch.cuda.synchronize()
            ev[0].record()
            out[k] = fn(*t)
            ev[1].record()
            torch.cuda.synchronize()
            if it >= warmup:
                times[k].append(ev[0].elapsed_time(ev[1]))
    return [(sorted(ts)[len(ts) // 2], min(ts), o) for ts, o in zip(times, out)]


def trace(fn, t):
    """(kernel launches, those of this library among them, device-to-host copies) of one step, by torch.profiler.
    `loss.backward()` itself launches one fill for its seed gradient, in both arms."""
    from torch.profiler import ProfilerActivity, profile
    fn(*t)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(*t)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    d2h = sum(1 for e in ev if "memcpy" in e.name.lower() and "dtoh" in e.name.lower())
    kernels = [e.name for e in ev if "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
    return len(kernels), sum(1 for k in kernels if "srcv" in k), d2h


def report(what, B, hw, info, ours, port, sets, steps, warmup):
    (ms, ms_min, (l_ours, g_ours)), (ms_port, ms_port_min, (l_port, g_port)) = timed([ours, port], sets, steps, warmup)
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
        "launches_port": k_port,
        "d2h_copies_ours": d2h_ours, "d2h_copies_port": d2h_port,
        "loss_ours": l_ours.item(), "loss_port": l_port.item(),
        "max_abs_grad_diff": (g_ours - g_port).abs().max().item(), "max_abs_grad": g_port.abs().max().item(),
        "grad_elements_differing_by_1e-3_of_max": int(((g_ours - g_port).abs() > 1e-3 * g_port.abs().max()).sum()),
        "grad_elements": g_port.numel(),
    }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 1])
    ap.add_argument("--height", type=int, default=192)
    ap.add_argument("--width", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gradloss.py needs a CUDA device")
    info = card()
    ms_ours, ms_port = step(S.MSGradientLoss()), step(O.ms_gradient_loss)
    si_ours, si_port = step(S.ScaleInvariantLoss(), (0, 1)), step(O.scale_invariant_loss, (0, 1))
    for B in a.batches:
        sets, si_sets = [], []
        for i in range(3):
            t = make_normals_batch(70 + i, B, a.height, a.width)
            gt, pred = t["depth_gt_b1hw"].cuda(), t["depth_pred_b1hw"].cuda()
            sets.append((gt, pred))
            n = B * a.height * a.width // 2
            lg = torch.log(pred.flatten()[:n]).contiguous()
            si_sets.append((lg + 0.05 * torch.randn_like(lg) + 0.02, lg))
        report("MSGradientLoss(gt, pred) + backward to pred", B, [a.height, a.width], info, ms_ours, ms_port, sets,
               a.steps, a.warmup)
        report("ScaleInvariantLoss on B H W / 2 elements + backward to both", B, [a.height, a.width], info, si_ours,
               si_port, si_sets, a.steps, a.warmup)


if __name__ == "__main__":
    main()
