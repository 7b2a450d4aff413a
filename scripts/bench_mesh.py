"""Timing + roofline of the marching-cubes mesh extraction (csrc/srcv_mesh.cuh, DESIGN §4.10), one JSON line.

    python scripts/bench_mesh.py [--steps 20] [--warmup 3]

Workloads, each after fusing the synthetic 6 x 5 x 3 m room from 8 depth maps of 240 x 320:
  full504  OurFuser's default volume without a ground-truth mesh: ±10 m at 4 cm = 504^3 voxels;
  room1cm  the room's own bounds at 1 cm: 608 x 512 x 312 voxels (as scripts/bench_tsdf.py).
Reported per workload and mode (single_mesh off / on):
  - ms per TSDF.extract_mesh (count + count read-back + extract), CUDA events over --steps warm calls;
  - ms of the count pass alone (srcv_mesh_count), and its algorithmic bandwidth: the values (plus the
    weights in single-mesh mode) read once;
  - V, F, and the algorithmic bytes of the whole extraction: the values (+ weights) read once per
    pass (4 passes over the volume: count, scan reads only block totals, vertices, faces -> 3) plus
    the outputs written -> GB/s and the fraction of the H100 SXM data-sheet 3.35 TB/s;
  - the reference's first step on the same volume, tsdf_values.cpu() (pageable host copy).
The reference's full host path (scikit-image marching_cubes) is not timed: scikit-image is not
available where this project runs.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402

import simplerecon_b200 as S  # noqa: E402
from simplerecon_b200 import _native  # noqa: E402
from simplerecon_b200.synthetic import make_tsdf_case  # noqa: E402

HBM_DATASHEET_GBS = 3350.0   # H100 SXM5 80 GB data sheet

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
a = ap.parse_args()


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:       # noqa: BLE001 - a missing tool only loses the annotation
        return None


def fused(bounds, voxel):
    c = make_tsdf_case(seed=21, frames=8, voxel_size=voxel, height=240, width=320, room=(6.0, 5.0, 3.0))
    vol = S.TSDF.from_bounds(bounds if bounds is not None else c["bounds"], voxel)
    S.TSDFFuser(vol, max_depth=3.0).integrate_depth(c["depth"].cuda(), c["cam_T_world"].cuda(), c["K"].cuda())
    torch.cuda.synchronize()
    return vol


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


def count_pass(vol, single):
    lib = _native.load()
    m = _native.MeshArgs()
    m.tsdf_values, m.tsdf_weights = vol.tsdf_values.data_ptr(), vol.tsdf_weights.data_ptr()
    m.X, m.Y, m.Z = vol.tsdf_values.shape
    m.voxel_size, m.scale_to_world, m.single_mesh = vol.voxel_size, 1, int(single)
    n = lib.srcv_mesh_workspace_bytes(C.byref(m))
    ws = torch.empty(n, dtype=torch.uint8, device="cuda")
    counts = torch.empty(2, dtype=torch.int64, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return lambda: _native.check(lib.srcv_mesh_count(C.byref(m), C.c_void_p(counts.data_ptr()),
                                                     C.c_void_p(ws.data_ptr()), n, stream))


def host_copy_ms(vol, reps=5):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        vol.tsdf_values.cpu()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


out = {"kernel": "tsdf_mesh_mc", "gpu": torch.cuda.get_device_name(), "power_limit_W": power_limit_w(),
       "steps": a.steps, "workloads": {}}
ten = {k: (-10.0 if k.endswith("min") else 10.0) for k in ("xmin", "xmax", "ymin", "ymax", "zmin", "zmax")}
for name, bounds, voxel in (("full504", ten, 0.04), ("room1cm", None, 0.01)):
    vol = fused(bounds, voxel)
    nvox = vol.tsdf_values.numel()
    w = {"volume": list(vol.tsdf_values.shape), "voxels": nvox, "values_MB": 2 * nvox / 1e6,
         "host_copy_ms": host_copy_ms(vol)}
    for single in (False, True):
        verts, faces, _ = vol.extract_mesh(single_mesh=single)
        V, F = len(verts), len(faces)
        del verts, faces
        ms = time_cuda(lambda: vol.extract_mesh(single_mesh=single), a.steps, a.warmup)
        cms = time_cuda(count_pass(vol, single), a.steps, a.warmup)
        in_bytes = (2 + (2 if single else 0)) * nvox
        alg = 3 * in_bytes + 24 * V + 12 * F
        w["single_mesh" if single else "default"] = {
            "V": V, "F": F, "ms_per_extract": ms, "faster_than_host_copy": ms < w["host_copy_ms"],
            "count_pass_ms": cms, "count_pass_GBps": in_bytes / (cms * 1e-3) / 1e9,
            "count_pass_frac_of_datasheet": in_bytes / (cms * 1e-3) / 1e9 / HBM_DATASHEET_GBS,
            "algorithmic_bytes": alg, "achieved_GBps": alg / (ms * 1e-3) / 1e9,
            "frac_of_datasheet": alg / (ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS}
    out["workloads"][name] = w
    del vol
    torch.cuda.empty_cache()
out["note"] = ("algorithmic bytes = values (+ weights in single-mesh mode) once per voxel pass (count, vertices, "
               "faces) + 24 B per vertex + 12 B per face; the reference's scikit-image host path is not timed "
               "(scikit-image is not available here)")
print(json.dumps(out))
