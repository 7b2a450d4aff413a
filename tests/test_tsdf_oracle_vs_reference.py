"""CPU: the TSDF oracle against the unmodified reference TSDFFuser (tools/tsdf.py), bit for bit in
fp16, after each of two integration rounds (stored outputs, tests/refgolden.py)."""
import pytest
import torch

from oracle import tsdf_oracle as T
from simplerecon_b200.synthetic import make_tsdf_case
from tests import refgolden

CASES = [(1, 1, 0.08, False), (2, 3, 0.05, False), (3, 2, 0.06, True)]
ROUNDS = 2               # the second round starts from non-trivial weights


def _case(seed, frames, voxel, masked):
    return make_tsdf_case(seed=seed, frames=frames, voxel_size=voxel, height=48, width=64, masked=masked)


def reference_outputs():
    """For tests/golden/make_reference_golden.py."""
    from oracle.ref_import import load_reference_tsdf
    R = load_reference_tsdf()
    out = {}
    for seed, frames, voxel, masked in CASES:
        c = _case(seed, frames, voxel, masked)
        ref = R.TSDF.from_bounds(c["bounds"], voxel_size=voxel)
        fuser = R.TSDFFuser(ref, max_depth=c["max_depth"], use_gpu=False)
        rec = {"min_depth": torch.tensor(fuser.min_depth)}
        for rep in range(ROUNDS):
            fuser.integrate_depth(c["depth"].half(), c["cam_T_world"].half(), c["K"].half(), c["mask"])
            rec[f"values{rep}"], rec[f"weights{rep}"] = ref.tsdf_values.clone(), ref.tsdf_weights.clone()
        out[f"{seed}_{frames}_{voxel}_{masked}"] = rec
    return out


@pytest.mark.parametrize("seed,frames,voxel,masked", CASES)
def test_integrate_matches_live_reference_bitwise(seed, frames, voxel, masked):
    G = refgolden.load("tsdf_oracle_vs_reference", f"{seed}_{frames}_{voxel}_{masked}")
    c = _case(seed, frames, voxel, masked)
    tv, tw, origin = T.new_volume(c["bounds"], voxel)
    assert tuple(tv.shape) == tuple(G["values0"].shape)
    # voxels whose fp16 sampling coordinate overflows: undefined in the CPU run of the reference
    # (see tsdf_oracle.overflow_voxels); a handful next to each camera's principal plane
    skip = T.overflow_voxels(origin, tuple(tv.shape), voxel, c["cam_T_world"], c["K"], c["depth"].shape[2:])
    assert skip.float().mean().item() < 1e-2
    keep = ~skip
    for rep in range(ROUNDS):
        rv, rw = G[f"values{rep}"], G[f"weights{rep}"]
        T.integrate(tv, tw, origin, voxel, c["depth"], c["cam_T_world"], c["K"], c["mask"],
                    min_depth=float(G["min_depth"]), max_depth=c["max_depth"])
        touched = int((rw > 0).sum())
        assert touched > 1000, touched
        assert torch.equal(tw[keep], rw[keep]), (tw.float() - rw.float())[keep].abs().max()
        assert torch.equal(tv[keep], rv[keep]), (tv.float() - rv.float())[keep].abs().max()
        # keep the two states identical for the next round (the skipped voxels differ by construction)
        tv[skip], tw[skip] = rv[skip], rw[skip]
