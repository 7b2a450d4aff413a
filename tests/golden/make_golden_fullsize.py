"""Golden vectors at the BENCH feature-map size (120 x 160, 7 views) from the UNMODIFIED reference.

    python tests/golden/make_golden_fullsize.py          (needs $SIMPLERECON_REF)

The fixtures of make_golden.py top out at 48 x 64, so they never reach the kernels' compile-time
160 x 120 instantiations.  At this size the inputs (8.6 MB of source features per frame) are too large
to commit: a case stores the generator call (simplerecon_b200.synthetic.make_tuple arguments), a SHA-256
of the regenerated inputs, and the reference classes' outputs — fp32, and the fp64 evaluation rounded
to fp32 together with max|ref32 - ref64| (what the parity bound needs).  tests/parity.py
`load_golden_fullsize` regenerates the inputs and refuses a hash mismatch.
"""
from __future__ import annotations

import hashlib
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from oracle.ref_import import load_reference  # noqa: E402
from simplerecon_b200.synthetic import make_tuple, mlp_state  # noqa: E402

OUT = Path(__file__).resolve().parent / "fullsize"
INPUT_KEYS = ("cur_feats", "src_feats", "src_extrinsics", "src_poses", "src_Ks", "cur_invK", "min_depth", "max_depth")


def inputs_sha256(tup) -> str:
    h = hashlib.sha256()
    for k in INPUT_KEYS:
        h.update(np.ascontiguousarray(tup[k].numpy()).tobytes())
    return h.hexdigest()


def run_case(R, name, kind, gen, D):
    tup = make_tuple(**gen)
    B, K, C, H, W = tup["src_feats"].shape
    sd = None
    if kind == "dot":
        mgr = R.CostVolumeManager(H, W, num_depth_bins=D)
    else:
        sd = mlp_state(K, C, seed=gen["seed"])
        mgr = R.FeatureVolumeManager(H, W, num_depth_bins=D, mlp_channels=[0, 128, 128, 1], matching_dim_size=C,
                                     num_source_views=K)
        mgr.load_state_dict({**mgr.state_dict(), **sd})
    with torch.no_grad():
        cost, lowest, planes, mask = mgr(**tup, return_mask=True)
        mgr64 = mgr.double()
        cost64, _, _, _ = mgr64(**{k: v.double() for k, v in tup.items()}, return_mask=True)
    err = float((cost.double() - cost64).abs().max())
    out = dict(kind=np.array(kind), D=np.array(D), gen=np.array(repr(sorted(gen.items()))), sha256=np.array(inputs_sha256(tup)),
               ref_cost=cost.numpy(), ref_cost64_as_f32=cost64.float().numpy(), err32v64=np.array(err),
               ref_lowest=lowest.numpy(), ref_planes=planes[:, :, 0, 0].numpy())
    if mask is not None:
        out["ref_mask"] = mask.numpy()
    OUT.mkdir(exist_ok=True)
    np.savez_compressed(OUT / f"{name}.npz", **out)
    print(f"{name}: cost {tuple(cost.shape)} max|c|={cost.abs().max():.4f} err32v64={err:.3e} sha {out['sha256']}")


if __name__ == "__main__":
    R = load_reference()
    gen = dict(batch=1, views=7, height=120, width=160, channels=16, seed=4321)
    run_case(R, "full_dot_120x160_D4_K7", "dot", gen, 4)
    run_case(R, "full_hero_120x160_D4_K7", "mlp", dict(gen, seed=4322), 4)
