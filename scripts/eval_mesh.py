"""Scores a predicted mesh or point cloud against a ground truth on the GPU (DESIGN §4.17).

    python scripts/eval_mesh.py PRED.ply GT.ply [--threshold 0.05] [--samples 1000000] [--seed 0]
                                [--views VIEWS.npz [--margin 0.05] [--max-depth D]] [--down-sample S] [--vertices]

Each PLY is binary little-endian (what ``TSDF.save``, ``SparseTSDF.save`` and ``ColorFuser.export_mesh``
write, or a ScanNet ``_vh_clean_2.ply``).  A file with faces is a mesh and is sampled uniformly by area
(``--samples`` points, seeded); a file without faces is a point cloud and is used as given.  Prints the six
metrics, one per line (metres for acc / comp / chamfer), then all of them as one JSON line.

With ``--views``, only the points of each side that the scan's depth frames observe are scored (DESIGN §4.18).
VIEWS.npz holds ``depths`` (F, H, W) float32 metres, ``K`` (4, 4) or (F, 4, 4) intrinsics at that resolution and
``cam_T_world`` (F, 4, 4) world -> camera.

With ``--down-sample S``, each side's points are voxel-down-sampled at voxel size S metres before scoring (DESIGN
§4.19; 0.02 approximates the 2 cm down-sampling NeuralRecon's evaluation is commonly run with).  With
``--vertices``, a file with faces is scored by its vertices, as a point cloud, instead of by surface samples.
"""
import argparse
import json
import math
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402

from simplerecon_b200.mesh_eval import DEFAULT_NUM_SAMPLES, Views, mesh_metrics  # noqa: E402
from simplerecon_b200.tsdf import read_ply  # noqa: E402


def side(path, vertices=False):
    verts, faces = read_ply(path)
    return (verts, faces) if faces is not None and len(faces) and not vertices else verts


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("pred")
    ap.add_argument("gt")
    ap.add_argument("--threshold", type=float, default=0.05, help="distance threshold of precision / recall, metres")
    ap.add_argument("--samples", type=int, default=DEFAULT_NUM_SAMPLES, help="samples drawn from each mesh")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--views", help="npz of depth frames (depths, K, cam_T_world): score only observed points")
    ap.add_argument("--margin", type=float, default=0.05, help="with --views: how far behind the depth a point may lie, metres")
    ap.add_argument("--max-depth", type=float, default=math.inf, help="with --views: the depth range of the frames, metres")
    ap.add_argument("--down-sample", type=float, default=None, help="voxel-down-sample both sides at this size, metres")
    ap.add_argument("--vertices", action="store_true", help="score a mesh file's vertices instead of surface samples")
    a = ap.parse_args(argv)
    views = None
    if a.views is not None:
        with np.load(a.views) as z:
            views = Views(z["depths"], z["K"], z["cam_T_world"], margin=a.margin, max_depth=a.max_depth)
    m = mesh_metrics(side(a.pred, a.vertices), side(a.gt, a.vertices), threshold=a.threshold, num_samples=a.samples,
                     seed=a.seed, views=views, down_sample=a.down_sample)
    for k, v in m.items():
        print(f"{k:10s} {v:.6f}")
    print(json.dumps(m))
    return m


if __name__ == "__main__":
    main()
