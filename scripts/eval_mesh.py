"""Scores a predicted mesh or point cloud against a ground truth on the GPU (DESIGN §4.17).

    python scripts/eval_mesh.py PRED.ply GT.ply [--threshold 0.05] [--samples 1000000] [--seed 0]

Each PLY is binary little-endian (what ``TSDF.save``, ``SparseTSDF.save`` and ``ColorFuser.export_mesh``
write, or a ScanNet ``_vh_clean_2.ply``).  A file with faces is a mesh and is sampled uniformly by area
(``--samples`` points, seeded); a file without faces is a point cloud and is used as given.  Prints the six
metrics, one per line (metres for acc / comp / chamfer), then all of them as one JSON line.
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from simplerecon_b200.mesh_eval import DEFAULT_NUM_SAMPLES, mesh_metrics  # noqa: E402
from simplerecon_b200.tsdf import read_ply  # noqa: E402


def side(path):
    verts, faces = read_ply(path)
    return (verts, faces) if faces is not None and len(faces) else verts


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("pred")
    ap.add_argument("gt")
    ap.add_argument("--threshold", type=float, default=0.05, help="distance threshold of precision / recall, metres")
    ap.add_argument("--samples", type=int, default=DEFAULT_NUM_SAMPLES, help="samples drawn from each mesh")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    m = mesh_metrics(side(a.pred), side(a.gt), threshold=a.threshold, num_samples=a.samples, seed=a.seed)
    for k, v in m.items():
        print(f"{k:10s} {v:.6f}")
    print(json.dumps(m))
    return m


if __name__ == "__main__":
    main()
