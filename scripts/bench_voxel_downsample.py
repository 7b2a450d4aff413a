"""Voxel down-sampling (DESIGN §4.19) on the GPU; one JSON line per workload.

    python scripts/bench_voxel_downsample.py [--rounds 5] [--frames 100] [--extreme-points 10000000]

Workloads:
  scene         process_scene's cloud (z_thresh 0.04, 3 consistent frames) of a synthetic scan from
                synthetic.make_mvs_scene, --frames frames at 480 x 640 of a 4 x 3 x 2.6 m room, with its uint8
                colours, down-sampled at 2 cm: the kernel, the numpy oracle (oracle/voxel_downsample_oracle.py, one
                round on the host) and the same rule as a PyTorch op sequence on the same GPU; then fuse_point_cloud
                against process_scene (host copies per frame) followed by voxel_down_sample.
  one_voxel     --extreme-points points in one 2 cm voxel: one thread walks them all (the kernel against the oracle).
  all_distinct  --extreme-points points, one per voxel, shuffled (the kernel, the oracle and the PyTorch sequence).
  mesh_metrics  DESIGN §4.17's slow case, process_scene's cloud of an 8-frame 240 x 320 scan against the room box
                (10^6 box samples), scored raw, with the cloud down-sampled at 2 cm, and with down_sample=0.02 on
                both sides.
Every arm's output is asserted bitwise equal to the kernel's.  Times are medians of --rounds, from a host clock
around whole calls that end in a device synchronise.  The card's name, power limit and max SM clock are read in the
same run with nvidia-smi queries.
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import simplerecon_b200 as S  # noqa: E402
from oracle import mesh_eval_oracle as O  # noqa: E402
from oracle import voxel_downsample_oracle as VD  # noqa: E402
from simplerecon_b200 import point_cloud_fusion as PCF  # noqa: E402
from simplerecon_b200.synthetic import make_mvs_scene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--frames", type=int, default=100)
ap.add_argument("--extreme-points", type=int, default=10_000_000)
ap.add_argument("--workloads", default="scene,one_voxel,all_distinct,mesh_metrics")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_voxel_downsample.py measures on a CUDA device; none found")
dev = torch.device("cuda")
ROOM = (4.0, 3.0, 2.6)


def smi(q):
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:       # noqa: BLE001 - a missing tool only loses the annotation
        return None


def timed(fn, rounds):
    out, ms = None, []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return out, ms


def same(x, y):
    """Bitwise equality of two (points, colours, counts) results, device or host."""
    for u, v in zip(x, y):
        if u is None or v is None:
            assert u is None and v is None
            continue
        u = u.cpu().numpy() if torch.is_tensor(u) else u
        v = v.cpu().numpy() if torch.is_tensor(v) else v
        assert u.shape == v.shape and np.array_equal(u.view(np.int32), v.view(np.int32)), "arms differ"


def arms(p, c, s, host=True, torch_arm=True):
    kern = lambda: PCF.voxel_down_sample(p, s, c)   # noqa: E731
    kern()
    res, t_k = timed(kern, a.rounds)
    out = {"points": len(p), "voxels": len(res[2]), "max_points_per_voxel": int(res[2].max()),
           "kernel_ms": statistics.median(t_k), "kernel_rounds_ms": t_k}
    if host:
        pn, cn = p.cpu().numpy(), (c.cpu().numpy() if c is not None else None)
        ref, t_h = timed(lambda: VD.voxel_down_sample(pn, s, cn), 1)
        same(res, ref)
        out.update(numpy_oracle_ms=t_h[0], speedup_vs_numpy=t_h[0] / out["kernel_ms"])
    if torch_arm:
        VD.voxel_down_sample_torch(p, s, c)
        ref, t_t = timed(lambda: VD.voxel_down_sample_torch(p, s, c), max(1, min(a.rounds, 3)))
        same(res, ref)
        out.update(torch_op_sequence_ms=statistics.median(t_t), torch_rounds_ms=t_t,
                   speedup_vs_torch=statistics.median(t_t) / out["kernel_ms"])
    return res, out


def box(size):
    v, f = O.box_mesh(size)
    return torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)


head = {"bench": "voxel_downsample", "gpu": torch.cuda.get_device_name(), "power_limit_W": smi("power.limit"),
        "clocks_max_sm_MHz": smi("clocks.max.sm"), "rounds": a.rounds}
work = a.workloads.split(",")
g = torch.Generator(device=dev).manual_seed(0)

if "scene" in work:
    sc = make_mvs_scene(seed=7, frames=a.frames, height=480, width=640, room=ROOM)
    d, im, E, K = (sc[k].to(dev) for k in ("depths", "images", "cam_T_world", "K"))
    (pts, rgb, _), t_ps = timed(lambda: PCF.process_scene(d, im, E, K, 0.04, 3), 1)
    p, c = torch.from_numpy(pts).to(dev), torch.from_numpy(rgb).to(dev)
    res, out = arms(p, c, 0.02)

    def host_path():
        hp, hc, _ = PCF.process_scene(d, im, E, K, 0.04, 3)
        return PCF.voxel_down_sample(hp, 0.02, hc)

    fused = lambda: S.fuse_point_cloud(d, im, E, K, z_thresh=0.04, n_consistent_thresh=3, voxel_size=0.02)  # noqa: E731
    fused()
    times = {"fuse": [], "host": []}
    for r in range(a.rounds):                          # alternating arms
        for k in (("fuse", "host") if r % 2 == 0 else ("host", "fuse")):
            got, ms = timed(fused if k == "fuse" else host_path, 1)
            same(got, res)
            times[k] += ms
    out.update(frames=a.frames, frame_hw=[480, 640], voxel_size=0.02, process_scene_ms=t_ps[0],
               fuse_point_cloud_ms=statistics.median(times["fuse"]), fuse_point_cloud_rounds_ms=times["fuse"],
               process_scene_then_down_sample_ms=statistics.median(times["host"]),
               process_scene_then_down_sample_rounds_ms=times["host"])
    print(json.dumps({**head, "workload": "scene", **out}), flush=True)
    del d, im, E, K, p, c, res

n = a.extreme_points
if "one_voxel" in work:
    p = 5.0 + torch.rand(n, 3, generator=g, device=dev) * 0.009
    _, out = arms(p, (torch.rand(n, 3, generator=g, device=dev) * 255).to(torch.uint8), 0.02, torch_arm=False)
    print(json.dumps({**head, "workload": "one_voxel", **out, "torch_op_sequence": "not run: one loop step per point"}),
          flush=True)

if "all_distinct" in work:
    side = int(np.ceil(n ** (1 / 3)))
    ar = torch.arange(side, device=dev, dtype=torch.float32)
    grid = torch.stack(torch.meshgrid(ar, ar, ar, indexing="ij"), -1).reshape(-1, 3)[:n]
    p = (grid * 0.03 + 0.01)[torch.randperm(len(grid), generator=g, device=dev)]
    _, out = arms(p, None, 0.02)
    print(json.dumps({**head, "workload": "all_distinct", **out}), flush=True)

if "mesh_metrics" in work:
    sc = make_mvs_scene(seed=21, frames=8, height=240, width=320, room=ROOM)
    d, im, E, K = (sc[k].to(dev) for k in ("depths", "images", "cam_T_world", "K"))
    raw = torch.from_numpy(PCF.process_scene(d, im, E, K, 0.1, 3)[0]).to(dev)
    ds = PCF.voxel_down_sample(raw, 0.02)[0]
    gt = box(ROOM)
    calls = {"raw": lambda: S.mesh_metrics(raw, gt, num_samples=1_000_000),
             "cloud_2cm": lambda: S.mesh_metrics(ds, gt, num_samples=1_000_000),
             "both_sides_down_sample_2cm": lambda: S.mesh_metrics(raw, gt, num_samples=1_000_000, down_sample=0.02)}
    out, res = {"cloud_points": len(raw), "cloud_2cm_points": len(ds)}, {}
    for k, fn in calls.items():
        fn()
        res[k], ms = timed(fn, a.rounds)
        out[f"{k}_ms"], out[f"{k}_rounds_ms"] = statistics.median(ms), ms
    print(json.dumps({**head, "workload": "mesh_metrics", **out, "metrics": res}), flush=True)
