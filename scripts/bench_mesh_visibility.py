"""Visibility-culled mesh evaluation (DESIGN §4.18) on the GPU; one JSON line per workload.

    python scripts/bench_mesh_visibility.py [--rounds 3] [--frames 300] [--workloads room_1e6,room_1e7]

Workload: scripts/bench_mesh_eval.py's synthetic 6 x 5 x 3 m room (240 x 320 depth, 4 batches of 8 frames fused
into a SparseTSDF at 2 cm, meshed with single_mesh=True) against the analytic room box, at 10^6 and 10^7 samples per
side, with two sets of views: "trajectory", --frames noise-free 480 x 640 depth maps of the box ray-cast
analytically along a loop through the room (positions on an ellipse at 1.1 - 1.7 m height, the view direction
swinging between the loop's tangent and the walls, pitched up and down: about the keyframes of one scan, seeing
more of the room than the fused frames did), and "fusion_frames", the 32 noisy 240 x 320 frames the prediction was
fused from, with the fuser's max_depth of 3 m (what test.py would pass).

Reported, medians of --rounds (CUDA-synchronised host clock around whole calls):
  - observation_counts on the ground-truth samples, with the per-tile frustum test and without it, and the same rule
    as a PyTorch op sequence on the same GPU (oracle/mesh_visibility_oracle.py); all three outputs are asserted equal;
  - (point, frame) pairs the kernel evaluated per point, with and without the tile test;
  - whole mesh_metrics calls with and without views, and the shares of each side's samples the views keep;
  - per direction and grid level the search statistics of DESIGN §4.17 on the culled sets;
  - the card's name, power limit and max SM clock, read in the same run (nvidia-smi queries only).
"""
import argparse
import json
import math
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import simplerecon_b200 as S  # noqa: E402
from oracle import mesh_visibility_oracle as VO  # noqa: E402
from simplerecon_b200 import mesh_eval as ME  # noqa: E402
from simplerecon_b200.synthetic import SCANNET_CX, SCANNET_CY, SCANNET_FX, SCANNET_FY, make_tsdf_case  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--frames", type=int, default=300)
ap.add_argument("--workloads", default="room_1e6,room_1e7")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_mesh_visibility.py measures on a CUDA device; none found")
dev = torch.device("cuda")
ROOM = (6.0, 5.0, 3.0)


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
    vol = S.SparseTSDF(0.02, max_blocks=1 << 17)
    fuser = S.TSDFFuser(vol, max_depth=3.0)
    cs = [make_tsdf_case(seed=200 + i, frames=8, voxel_size=0.02, height=240, width=320, room=ROOM) for i in range(4)]
    for c in cs:
        fuser.integrate_depth(c["depth"].to(dev), c["cam_T_world"].to(dev), c["K"].to(dev))
    verts, faces, _ = vol.extract_mesh(single_mesh=True)
    fusion_views = S.Views(*(torch.cat([c[k] for c in cs]).to(dev) for k in ("depth", "K", "cam_T_world")),
                           margin=0.05, max_depth=3.0)
    return (verts, faces), box(ROOM), fusion_views


def look_at(pos, fwd):
    """world -> camera (4, 4) fp64 of a camera at pos looking along fwd, x right and y down, world z up."""
    z = fwd / np.linalg.norm(fwd)
    x = np.cross(z, [0.0, 0.0, 1.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    E = np.eye(4)
    E[:3, :3] = np.stack([x, y, z])
    E[:3, 3] = -E[:3, :3] @ pos
    return E


def scan_views(frames, H=480, W=640):
    """``frames`` ray-cast depth maps of the room box along a loop through the room; (depths, K, cam_T_world)."""
    K = np.eye(4)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = SCANNET_FX * W / 640, SCANNET_FY * H / 480, SCANNET_CX * W / 640, \
        SCANNET_CY * H / 480
    c = np.asarray(ROOM) / 2
    Es = []
    for i in range(frames):
        s = 2 * math.pi * i / frames
        pos = c + [1.6 * math.cos(s), 1.3 * math.sin(s), 0.3 * math.sin(3 * s) - 0.2]
        tangent = np.array([-math.sin(s), math.cos(s), 0.0])
        outward = np.array([math.cos(s), math.sin(s), 0.0])
        sw = math.sin(5 * s)
        fwd = tangent * math.cos(sw) + outward * math.sin(sw) + [0.0, 0.0, 0.35 * math.sin(7 * s)]
        Es.append(look_at(pos, fwd))
    E = torch.tensor(np.stack(Es), dtype=torch.float64, device=dev)
    Kt = torch.tensor(K, dtype=torch.float64, device=dev)
    v, u = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev) + 0.5,
                          torch.arange(W, dtype=torch.float64, device=dev) + 0.5, indexing="ij")
    rays = torch.stack([(u - Kt[0, 2]) / Kt[0, 0], (v - Kt[1, 2]) / Kt[1, 1], torch.ones_like(u)], -1)   # z = 1
    hi = torch.tensor(ROOM, dtype=torch.float64, device=dev)
    depths = torch.empty(frames, H, W, dtype=torch.float32, device=dev)
    for f in range(frames):
        R = E[f, :3, :3]
        pos = -R.T @ E[f, :3, 3]
        d = rays @ R                                                       # world directions
        t = torch.where(d > 0, (hi - pos) / d.clamp_min(1e-12), -pos / d.clamp_max(-1e-12))
        depths[f] = t.min(-1).values.float()
    return depths, Kt.float(), E.float()


def timed(fn, rounds):
    out, ms = None, []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return out, ms


def search_stats(q, t):
    st = torch.zeros(8, dtype=torch.int64, device=dev)
    ME._distances(q, t, torch.zeros(1, dtype=torch.int32, device=dev), st)
    st = st.tolist()
    return {"queries": len(q), "targets": len(t), "candidates_per_query_by_level": [c / len(q) for c in st[:4]],
            "open_share_by_level": [o / len(q) for o in st[4:]], "brute_force_share": st[7] / len(q)}


def workload(pred, gt, views, n, seed=0, tau=0.05):
    d, K, E = views[:3]
    P, G = ME.sample_surface(*pred, n, seed=seed), ME.sample_surface(*gt, n, seed=seed + 1)
    count = lambda cull, st=None: ME._observation_counts(G, d, K, E, views.margin, views.max_depth,   # noqa: E731
                                                         tile_cull=cull, stats=st)
    count(True), count(False)
    c_cull, t_cull = timed(lambda: count(True), a.rounds)
    c_all, t_all = timed(lambda: count(False), a.rounds)
    c_torch, t_torch = timed(lambda: VO.observation_counts_torch(G, d, K, E, views.margin, views.max_depth),
                             max(1, min(a.rounds, 2)))
    assert torch.equal(c_cull, c_all) and torch.equal(c_cull, c_torch), "observation counts differ"
    tested = {}
    for name, cull in (("tile_test", True), ("every_frame", False)):
        st = torch.zeros(1, dtype=torch.int64, device=dev)
        count(cull, st)
        tested[name] = int(st) / n
    full = lambda: ME.mesh_metrics(pred, gt, threshold=tau, num_samples=n, seed=seed)   # noqa: E731
    culled = lambda: ME.mesh_metrics(pred, gt, threshold=tau, num_samples=n, seed=seed, views=views)   # noqa: E731
    full(), culled()
    times = {"full": [], "culled": []}
    res = {}
    for r in range(a.rounds):                         # alternating arms
        for k in (("full", "culled") if r % 2 == 0 else ("culled", "full")):
            res[k], ms = timed(full if k == "full" else culled, 1)
            times[k] += ms
            print(f"n={n} round {r} {k}: {ms[0]:.1f} ms", file=sys.stderr, flush=True)
    cP = ME._observation_counts(P, d, K, E, views.margin, views.max_depth)
    Pk, Gk = P[cP > 0], G[c_cull > 0]
    return {"samples_per_mesh": n, "frames": len(d), "frame_hw": list(d.shape[-2:]), "max_depth": views.max_depth,
            "observation_counts_ms": statistics.median(t_cull), "observation_counts_rounds_ms": t_cull,
            "observation_counts_no_tile_test_ms": statistics.median(t_all),
            "torch_op_sequence_ms": statistics.median(t_torch), "torch_rounds_ms": t_torch,
            "speedup_vs_torch": statistics.median(t_torch) / statistics.median(t_cull),
            "frames_tested_per_point": tested,
            "gt_kept_share": len(Gk) / n, "pred_kept_share": len(Pk) / n,
            "mesh_metrics_ms": statistics.median(times["full"]), "mesh_metrics_rounds_ms": times["full"],
            "mesh_metrics_views_ms": statistics.median(times["culled"]), "mesh_metrics_views_rounds_ms": times["culled"],
            "metrics": res["full"], "metrics_views": res["culled"],
            "search_culled": {"pred_to_gt": search_stats(Pk, Gk), "gt_to_pred": search_stats(Gk, Pk)},
            "search_full": {"gt_to_pred": search_stats(G, P)}}


head = {"bench": "mesh_visibility", "gpu": torch.cuda.get_device_name(), "power_limit_W": smi("power.limit"),
        "clocks_max_sm_MHz": smi("clocks.max.sm"), "rounds": a.rounds}
room_mesh, room_box, fusion_views = fused_room()
all_views = (("trajectory", S.Views(*scan_views(a.frames), margin=0.05)), ("fusion_frames", fusion_views))
for name, n in (("room_1e6", 1_000_000), ("room_1e7", 10_000_000)):
    if name in a.workloads.split(","):
        for vname, views in all_views:
            out = workload(room_mesh, room_box, views, n)
            print(json.dumps({**head, "workload": name, "views": vname, "room_mesh_faces": int(len(room_mesh[1])), **out}),
                  flush=True)
