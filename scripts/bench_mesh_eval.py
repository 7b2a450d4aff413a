"""GPU mesh evaluation (DESIGN §4.17) against scipy's cKDTree on the host, on the same points; one JSON line.

    python scripts/bench_mesh_eval.py [--rounds 3] [--host-rounds N] [--workloads room_1e6,room_1e7,pointcloud]

Workloads:
  room_1e6     the synthetic 6 x 5 x 3 m room of scripts/bench_tsdf_sparse.py (240 x 320 depth, 4 batches of 8
               frames) fused into a SparseTSDF at 2 cm, meshed with single_mesh=True, against the analytic room
               box, 10^6 samples per side;
  room_1e7     the same at 10^7 samples per side;
  pointcloud   process_scene's point cloud of an 8-frame 240 x 320 scan of a 4 x 3 x 2.6 m room against the box
               (10^6 box samples).
GPU: simplerecon_b200.mesh_metrics per call (sampling included).  Host: the same sample sets, copied to the
host once, scored with cKDTree(...).query(workers=-1) in both directions (tree builds included) and numpy
means.  The two are timed in alternating rounds (the host arm in the first --host-rounds of them, default all)
and the medians reported, with both results (they agree to rounding), the peak device memory of one GPU call, and
per direction and grid level the target points the search evaluated per query and the share of queries the level
left open (the last level's share went to the brute force).  One JSON line per workload, printed as soon as it is
done, each with the card's name, power limit and max SM clock read in the same run (nvidia-smi queries only).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.spatial import cKDTree  # noqa: E402

import simplerecon_b200 as S  # noqa: E402
from simplerecon_b200 import mesh_eval as ME, point_cloud_fusion as pcf  # noqa: E402
from simplerecon_b200.synthetic import make_mvs_scene, make_tsdf_case  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--host-rounds", type=int, default=None, help="rounds with the host arm (default: all)")
ap.add_argument("--workloads", default="room_1e6,room_1e7,pointcloud")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_mesh_eval.py measures on a CUDA device; none found")
dev = torch.device("cuda")


def smi(q):
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:       # noqa: BLE001 - a missing tool only loses the annotation
        return None


def box(size):
    s = np.asarray(size, np.float32)
    v = np.array([[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)], np.float32) * s
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for q0, q1, q2, q3 in quads for t in ((q0, q1, q2), (q0, q2, q3))], np.int32)
    return torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)


def fused_room():
    room = (6.0, 5.0, 3.0)
    vol = S.SparseTSDF(0.02, max_blocks=1 << 17)
    fuser = S.TSDFFuser(vol, max_depth=3.0)
    for i in range(4):
        c = make_tsdf_case(seed=200 + i, frames=8, voxel_size=0.02, height=240, width=320, room=room)
        fuser.integrate_depth(c["depth"].to(dev), c["cam_T_world"].to(dev), c["K"].to(dev))
    verts, faces, _ = vol.extract_mesh(single_mesh=True)
    return (verts, faces), box(room)


def scene_cloud():
    room = (4.0, 3.0, 2.6)
    sc = make_mvs_scene(seed=21, frames=8, height=240, width=320, room=room)
    d, im, P, K = (sc[k].to(dev) for k in ("depths", "images", "cam_T_world", "K"))
    pts, _, _ = pcf.process_scene(d, im, P, K, 0.1, 3)
    return torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32)).to(dev), box(room)


def host_metrics(P, G, tau):
    dp = cKDTree(G).query(P, k=1, workers=-1)[0]
    dg = cKDTree(P).query(G, k=1, workers=-1)[0]
    acc, comp = float(dp.mean()), float(dg.mean())
    pr, rc = float(np.count_nonzero(dp < tau)) / len(dp), float(np.count_nonzero(dg < tau)) / len(dg)
    return dict(zip(ME.KEYS, (acc, comp, (acc + comp) / 2, pr, rc, 2 * pr * rc / (pr + rc) if pr + rc else 0.0)))


def workload(pred, gt, n, seed=0, tau=0.05):
    gpu = lambda: ME.mesh_metrics(pred, gt, threshold=tau, num_samples=n, seed=seed)   # noqa: E731
    side = lambda x, s: ME.sample_surface(*x, n, seed=s) if isinstance(x, tuple) else x   # noqa: E731
    P, G = side(pred, seed), side(gt, seed + 1)
    Ph, Gh = (t.cpu().numpy().astype(np.float64) for t in (P, G))
    gpu()
    torch.cuda.synchronize()
    times = {"gpu": [], "host": []}
    res = {}
    for r in range(a.rounds):
        arms = ("gpu", "host") if r % 2 == 0 else ("host", "gpu")
        for k in (arms if a.host_rounds is None or r < a.host_rounds else ("gpu",)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[k] = gpu() if k == "gpu" else host_metrics(Ph, Gh, tau)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
            print(f"n={n} round {r} {k}: {times[k][-1]:.1f} ms", file=sys.stderr, flush=True)
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    gpu()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    stats = {}
    for name, q, t in (("pred_to_gt", P, G), ("gt_to_pred", G, P)):
        st = torch.zeros(8, dtype=torch.int64, device=dev)
        ME._distances(q, t, torch.zeros(1, dtype=torch.int32, device=dev), st)
        st = st.tolist()
        stats[name] = {"queries": len(q), "targets": len(t),
                       "candidates_per_query_by_level": [c / len(q) for c in st[:4]],
                       "open_share_by_level": [o / len(q) for o in st[4:]], "brute_force_share": st[7] / len(q)}
    out = {"samples_per_mesh": n, "pred_points": len(P), "gt_points": len(G),
           "gpu_ms": statistics.median(times["gpu"]), "gpu_rounds_ms": times["gpu"],
           "host_ckdtree_ms": statistics.median(times["host"]), "host_rounds_ms": times["host"],
           "gpu_peak_MB": peak / 2 ** 20, "search": stats, "gpu_metrics": res["gpu"], "host_metrics": res["host"],
           "max_rel_diff": max(abs(res["gpu"][k] - res["host"][k]) / max(abs(res["host"][k]), 1e-300) for k in ME.KEYS)}
    out["speedup"] = out["host_ckdtree_ms"] / out["gpu_ms"]
    return out


head = {"bench": "mesh_eval", "gpu": torch.cuda.get_device_name(), "power_limit_W": smi("power.limit"),
        "clocks_max_sm_MHz": smi("clocks.max.sm"), "host_cpus": os.cpu_count(), "rounds": a.rounds,
        "host_rounds": a.host_rounds if a.host_rounds is not None else a.rounds}


def report(name, out, **extra):
    print(json.dumps({**head, "workload": name, **extra, **out}), flush=True)


wanted = a.workloads.split(",")
if "room_1e6" in wanted or "room_1e7" in wanted:
    room_mesh, room_box = fused_room()
    for name, n in (("room_1e6", 1_000_000), ("room_1e7", 10_000_000)):
        if name in wanted:
            report(name, workload(room_mesh, room_box, n), room_mesh_faces=int(len(room_mesh[1])))
if "pointcloud" in wanted:
    cloud, cloud_box = scene_cloud()
    report("pointcloud", workload(cloud, cloud_box, 1_000_000))
