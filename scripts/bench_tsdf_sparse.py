"""Dense vs voxel-block TSDF fusion (DESIGN §4.16), one JSON line.

    python scripts/bench_tsdf_sparse.py [--steps 10] [--warmup 2] [--rounds 3]

The synthetic 6 x 5 x 3 m room of scripts/bench_color_fusion.py (depth maps of 240 x 320, 8 frames per
integrate_depth call, 4 seeded batches in turn), max_depth 3 m:
  4cm / 2cm   the ±10 m cube the reference allocates without a ground-truth mesh (504^3 and 1000^3 voxels)
              against SparseTSDF on the same lattice;
  1cm         the room's own bounds (what a ground-truth mesh gives, 608 x 512 x 312 voxels) against
              SparseTSDF on that lattice.
Per workload: integration ms per call and per frame (dense and sparse timed in alternating rounds, the
median of the rounds reported), extract_mesh ms (median of the rounds), peak device memory of building
the volume, one call and one mesh (torch.cuda.max_memory_allocated), and the blocks allocated.  The
volumes' values and weights are compared after the timed calls (to_dense over the dense volume's box).
The card's name, power limit and max SM clock are read in the same run (nvidia-smi queries only).
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402

import simplerecon_b200 as S  # noqa: E402
from simplerecon_b200.synthetic import make_tsdf_case  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--rounds", type=int, default=3)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_tsdf_sparse.py measures on a CUDA device; none found")

ROOM = (6.0, 5.0, 3.0)
FRAMES = 8


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


cases = []
for i in range(4):
    c = make_tsdf_case(seed=200 + i, frames=FRAMES, voxel_size=0.04, height=240, width=320, room=ROOM)
    cases.append({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()})
TEN = {k: (-10.0 if k.endswith("min") else 10.0) for k in ("xmin", "xmax", "ymin", "ymax", "zmin", "zmax")}
ROOM_BOUNDS = {"xmin": -0.04, "xmax": ROOM[0] + 0.04, "ymin": -0.04, "ymax": ROOM[1] + 0.04, "zmin": -0.04,
               "zmax": ROOM[2] + 0.04}


def make(kind, bounds, voxel, max_blocks):
    if kind == "dense":
        return S.TSDF.from_bounds(bounds, voxel)
    return S.SparseTSDF.from_bounds(bounds, voxel, max_blocks=max_blocks)


def stepper(fuser):
    it = iter(range(1 << 30))

    def step():
        d = cases[next(it) % 4]
        fuser.integrate_depth(d["depth"], d["cam_T_world"], d["K"])
    return step


def peak_memory(kind, bounds, voxel, max_blocks):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    vol = make(kind, bounds, voxel, max_blocks)
    stepper(S.TSDFFuser(vol, max_depth=3.0))()
    vol.extract_mesh()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del vol
    torch.cuda.empty_cache()
    return peak


def workload(bounds, voxel, max_blocks):
    vols = {k: make(k, bounds, voxel, max_blocks) for k in ("dense", "sparse")}
    steps = {k: stepper(S.TSDFFuser(v, max_depth=3.0)) for k, v in vols.items()}
    integ = {k: [] for k in vols}
    mesh = {k: [] for k in vols}
    for r in range(a.rounds):                 # alternating, paired rounds
        for k in (("dense", "sparse") if r % 2 == 0 else ("sparse", "dense")):
            integ[k].append(time_cuda(steps[k], a.steps, a.warmup))
            mesh[k].append(time_cuda(lambda: vols[k].extract_mesh(), 2, 1))
    dense, sparse = vols["dense"], vols["sparse"]
    back = sparse.to_dense(bounds)
    equal = bool(torch.equal(back.tsdf_values.view(torch.int16), dense.tsdf_values.view(torch.int16)) and
                 torch.equal(back.tsdf_weights.view(torch.int16), dense.tsdf_weights.view(torch.int16)))
    blocks = sparse.allocated_blocks
    F = {k: int(len(v.extract_mesh()[1])) for k, v in vols.items()}
    del back, vols, steps, dense, sparse
    torch.cuda.empty_cache()
    out = {"voxel_m": voxel, "max_blocks": max_blocks, "allocated_blocks": blocks,
           "allocated_block_MB": blocks * 512 * 4 / 2 ** 20, "values_weights_equal": equal, "faces": F}
    for k in ("dense", "sparse"):
        ms = statistics.median(integ[k])
        out[k] = {"integrate_ms_per_call": ms, "integrate_ms_per_frame": ms / FRAMES, "integrate_rounds_ms": integ[k],
                  "mesh_ms": statistics.median(mesh[k]), "mesh_rounds_ms": mesh[k],
                  "peak_MB": peak_memory(k, bounds, voxel, max_blocks) / 2 ** 20}
    out["integrate_speedup"] = out["dense"]["integrate_ms_per_call"] / out["sparse"]["integrate_ms_per_call"]
    out["mesh_speedup"] = out["dense"]["mesh_ms"] / out["sparse"]["mesh_ms"]
    return out


res = {"bench": "tsdf_sparse", "gpu": torch.cuda.get_device_name(), "power_limit_W": smi("power.limit"),
       "clocks_max_sm_MHz": smi("clocks.max.sm"), "steps": a.steps, "rounds": a.rounds, "frames_per_call": FRAMES,
       "depth_hw": [240, 320], "workloads": {}}
for name, bounds, voxel, mb in (("cube_4cm", TEN, 0.04, 1 << 16), ("cube_2cm", TEN, 0.02, 1 << 17),
                                ("room_1cm", ROOM_BOUNDS, 0.01, 1 << 19)):
    res["workloads"][name] = workload(bounds, voxel, mb)
print(json.dumps(res))
