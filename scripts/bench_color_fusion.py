"""What colour costs in the kernel-backed TSDF (DESIGN §4.11), plain vs colour, one JSON line.

    python scripts/bench_color_fusion.py [--steps 20] [--warmup 3]

Workloads (the synthetic 6 x 5 x 3 m room, depth maps of 240 x 320, colour frames of 480 x 640):
  room1cm  the room's bounds at 1 cm (as scripts/bench_tsdf.py), full504  ±10 m at 4 cm = 504^3 voxels;
  integration of 1 and of 8 frames per call: ms per call, plain and colour; algorithmic bytes = 8 B per
    updated voxel (plain) and + 24 B (colour planes read and written) -> GB/s;
  extract_mesh, plain vs with_colors, on the volume fused from 8 frames: ms per call;
  live meshing: per frame, 1 frame of 192 x 256 fused with its colour, the coloured mesh extracted and a
    PLY written (4 cm room, 10 frames): ms per frame, host write included.
Clocks and the power limit are read in the same run (nvidia-smi queries only).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402

import simplerecon_b200 as S  # noqa: E402
from simplerecon_b200.synthetic import make_color_tsdf_case  # noqa: E402
from simplerecon_b200.tsdf import colors_to_u8, write_ply  # noqa: E402

HBM_DATASHEET_GBS = 3350.0   # H100 SXM5 80 GB data sheet

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
a = ap.parse_args()


def smi(q):
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:       # noqa: BLE001 - a missing tool only loses the annotation
        return None


def time_cuda(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def cases(frames):
    out = []
    for i in range(4):
        c = make_color_tsdf_case(seed=100 + i, frames=frames, voxel_size=0.04, height=240, width=320,
                                 color_hw=(480, 640), room=(6.0, 5.0, 3.0))
        out.append({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()})
    return out


def integration(bounds, voxel, frames):
    cs = cases(frames)
    res = {}
    for color in (False, True):
        vol = S.TSDF.from_bounds(bounds, voxel, color=color)
        fuser = S.TSDFFuser(vol, max_depth=3.0)
        it = iter(range(1 << 30))

        def step():
            d = cs[next(it) % 4]
            fuser.integrate_depth(d["depth"], d["cam_T_world"], d["K"], color_b3hw=d["color"] if color else None)
        res["color" if color else "plain"] = {"ms_per_call": time_cuda(step, a.steps, a.warmup)}
        del vol, fuser
        torch.cuda.empty_cache()
    touched = []
    for d in cs:      # voxels one call updates, on a fresh volume
        v0 = S.TSDF.from_bounds(bounds, voxel)
        S.TSDFFuser(v0, max_depth=3.0).integrate_depth(d["depth"], d["cam_T_world"], d["K"])
        touched.append(int((v0.tsdf_weights > 0).sum()))
        del v0
    t = sum(touched) / len(touched)
    for k, per in (("plain", 8), ("color", 32)):
        r = res[k]
        r["algorithmic_bytes"] = per * t
        r["GBps"] = per * t / (r["ms_per_call"] * 1e-3) / 1e9
        r["frac_of_datasheet"] = r["GBps"] / HBM_DATASHEET_GBS
    res["updated_voxels_per_call"] = t
    res["color_overhead"] = res["color"]["ms_per_call"] / res["plain"]["ms_per_call"]
    return res


def mesh(bounds, voxel):
    c = cases(8)[0]
    vol = S.TSDF.from_bounds(bounds, voxel, color=True)
    S.TSDFFuser(vol, max_depth=3.0).integrate_depth(c["depth"], c["cam_T_world"], c["K"], color_b3hw=c["color"])
    V = len(vol.extract_mesh()[0])
    plain = time_cuda(lambda: vol.extract_mesh(), a.steps, a.warmup)
    colored = time_cuda(lambda: vol.extract_mesh(with_colors=True), a.steps, a.warmup)
    return {"volume": list(vol.tsdf_values.shape), "V": V, "plain_ms": plain, "with_colors_ms": colored,
            "color_overhead": colored / plain}


def live(out_dir):
    c = make_color_tsdf_case(seed=7, frames=10, voxel_size=0.04, height=192, width=256, color_hw=(192, 256),
                             room=(6.0, 5.0, 3.0))
    g = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()}
    fuser = S.ColorFuser(gt_path=None, fusion_resolution=0.04, max_fusion_depth=3.0)
    vol = S.TSDF.from_bounds(c["bounds"], 0.04, color=True)
    fuser.tsdf_fuser_pred = S.TSDFFuser(vol, max_depth=3.0)       # the room's bounds instead of ±10 m
    path = os.path.join(out_dir, "live.ply")
    ts = []
    for b in range(10):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fuser.fuse_frames(g["depth"][b:b + 1], g["K"][b:b + 1], g["cam_T_world"][b:b + 1], g["color"][b:b + 1])
        fuser.export_mesh(path)
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"frames": 10, "ms_per_frame_median": sorted(ts[2:])[len(ts[2:]) // 2], "ms_per_frame_all": ts,
            "ply_bytes": os.path.getsize(path)}


ten = {k: (-10.0 if k.endswith("min") else 10.0) for k in ("xmin", "xmax", "ymin", "ymax", "zmin", "zmax")}
room = make_color_tsdf_case(seed=100, frames=1, voxel_size=0.01, height=8, width=8, color_hw=(8, 8),
                            room=(6.0, 5.0, 3.0))["bounds"]
out = {"bench": "color_fusion", "gpu": torch.cuda.get_device_name(), "power_limit_W": smi("power.limit"),
       "clocks_max_sm_MHz": smi("clocks.max.sm"), "steps": a.steps, "integration": {}, "extract_mesh": {}}
for name, bounds, voxel in (("room1cm", room, 0.01), ("full504", ten, 0.04)):
    for frames in (1, 8):
        out["integration"][f"{name}_{frames}f"] = integration(bounds, voxel, frames)
    out["extract_mesh"][name] = mesh(bounds, voxel)
    torch.cuda.empty_cache()
with tempfile.TemporaryDirectory() as d:
    out["live_meshing_4cm"] = live(d)
out["clocks_sm_MHz_after"] = smi("clocks.sm")
print(json.dumps(out))
