"""CPU: the oracle against the outputs of the unmodified reference classes on randomised shapes
(stored under tests/golden/reference/, see tests/refgolden.py)."""
import pytest
import torch

from oracle import costvolume_oracle as O
from simplerecon_b200.synthetic import make_tuple, mlp_state
from tests import refgolden
from tests.parity import assert_cost_close

DOT_CASES = [(2, 3, 20, 28, 6, 1), (1, 7, 15, 21, 5, 2), (3, 1, 8, 8, 3, 3)]
MLP_CASES = [(2, 3, 12, 16, 4, 4), (1, 7, 10, 14, 3, 5)]
GRAD_CASE = (2, 3, 10, 14, 4, 17)
RANGE_CASE = (3, 2, 10, 12, 5, 31)


def _name(kind, case):
    return kind + "_" + "_".join(map(str, case))


def _golden(kind, case=()):
    return refgolden.load("oracle_vs_reference", _name(kind, case))


def _grad_tuple():
    B, K, H, W, D, seed = GRAD_CASE
    return make_tuple(B, K, H, W, seed=seed), torch.randn(B, D, H, W, generator=torch.Generator().manual_seed(1))


def _range_tuple():
    B, K, H, W, D, seed = RANGE_CASE
    t = make_tuple(B, K, H, W, seed=seed)
    t["min_depth"] = torch.tensor([0.25, 0.5, 0.3]).view(B, 1, 1, 1)
    t["max_depth"] = torch.tensor([5.0, 8.0, 2.0]).view(B, 1, 1, 1)
    return t


def reference_outputs():
    """For tests/golden/make_reference_golden.py."""
    from oracle.ref_import import load_reference
    R = load_reference()
    out = {}
    with torch.no_grad():
        for B, K, H, W, D, seed in DOT_CASES:
            rc, rl, rp, rm = R.CostVolumeManager(H, W, num_depth_bins=D)(**make_tuple(B, K, H, W, seed=seed))
            assert rm is None
            out[_name("dot", (B, K, H, W, D, seed))] = dict(cost=rc, lowest=rl, planes=rp.contiguous())
        for B, K, H, W, D, seed in MLP_CASES:
            t = make_tuple(B, K, H, W, seed=seed)
            ref = R.FeatureVolumeManager(H, W, num_depth_bins=D, mlp_channels=[0, 128, 128, 1],
                                         matching_dim_size=16, num_source_views=K)
            ref.load_state_dict({**ref.state_dict(), **mlp_state(K, 16, seed=seed)})
            rc, rl, rp, rm = ref(**t, return_mask=True)
            fc, fl, fp, fm = ref.to_fast()(**t, return_mask=True)
            out[_name("mlp", (B, K, H, W, D, seed))] = dict(cost=rc, lowest=rl, mask=rm, fast_cost=fc, fast_mask=fm)
        rc, rr, rt = R.pose_distance(make_tuple(3, 5, 4, 4, seed=9)["src_poses"].reshape(-1, 4, 4))
        out[_name("pose", ())] = dict(comb=rc, r=rr, t=rt)
        B, K, H, W, D, seed = RANGE_CASE
        rc, rl, rp, _ = R.CostVolumeManager(H, W, num_depth_bins=D)(**_range_tuple())
        out[_name("range", RANGE_CASE)] = dict(cost=rc, lowest=rl, planes=rp.contiguous())
    B, K, H, W, D, seed = GRAD_CASE
    t, g = _grad_tuple()
    t["cur_feats"] = t["cur_feats"].clone().requires_grad_(True)
    t["src_feats"] = t["src_feats"].clone().requires_grad_(True)
    cost, *_ = R.CostVolumeManager(H, W, num_depth_bins=D)(**t)
    (cost * g).sum().backward()
    out[_name("grad", GRAD_CASE)] = dict(gcur=t["cur_feats"].grad, gsrc=t["src_feats"].grad)
    return out


@pytest.mark.parametrize("B,K,H,W,D,seed", DOT_CASES)
def test_dot_matches_live_reference(B, K, H, W, D, seed):
    G = _golden("dot", (B, K, H, W, D, seed))
    t = make_tuple(B, K, H, W, seed=seed)
    oc, ol, op, om = O.forward_dot(**t, num_depth_bins=D, sampler="aten")
    assert torch.equal(op.contiguous(), G["planes"])
    assert (oc - G["cost"]).abs().max().item() <= 2e-6 * float(G["cost"].abs().max())
    assert torch.equal(ol, G["lowest"]) and om is None
    oc2, *_ = O.forward_dot(**t, num_depth_bins=D, sampler="explicit")
    assert_cost_close("dot", oc2, G["cost"])


@pytest.mark.parametrize("B,K,H,W,D,seed", MLP_CASES)
def test_mlp_matches_live_reference_slow_and_fast(B, K, H, W, D, seed):
    G = _golden("mlp", (B, K, H, W, D, seed))
    t = make_tuple(B, K, H, W, seed=seed)
    w = O.mlp_weights_from_state_dict(mlp_state(K, 16, seed=seed))
    oc, ol, op, om = O.forward_mlp(**t, weights=w, num_depth_bins=D, return_mask=True, sampler="aten")
    for c in (G["cost"], G["fast_cost"]):
        assert (oc - c).abs().max().item() <= 5e-6 * float(c.abs().max()) + 1e-7
    assert torch.equal(om, G["mask"]) and torch.equal(om, G["fast_mask"])
    assert torch.equal(ol, G["lowest"])


def test_pose_distance_matches_live_reference():
    G = _golden("pose")
    comb, r, tm = O.pose_distance(make_tuple(3, 5, 4, 4, seed=9)["src_poses"])
    assert torch.allclose(comb.reshape(-1), G["comb"]) and torch.allclose(r.reshape(-1), G["r"])
    assert torch.allclose(tm.reshape(-1), G["t"])


def test_dot_gradients_match_live_reference_autograd():
    """The oracle's autograd (which the GPU backward kernel is tested against) equals autograd
    through the reference's own CostVolumeManager for the two feature inputs."""
    G = _golden("grad", GRAD_CASE)
    D = GRAD_CASE[4]
    t, g = _grad_tuple()
    t["cur_feats"] = t["cur_feats"].clone().requires_grad_(True)
    t["src_feats"] = t["src_feats"].clone().requires_grad_(True)
    cost, *_ = O.forward_dot(**t, num_depth_bins=D, sampler="explicit")
    (cost * g).sum().backward()
    for a, b in ((G["gcur"], t["cur_feats"].grad), (G["gsrc"], t["src_feats"].grad)):
        assert (a - b).abs().max().item() <= 2e-5 * float(a.abs().max()) + 1e-6


def test_per_frame_depth_range_matches_live_reference():
    """(B,1,1,1) min/max depth: the reference's generate_depth_planes broadcasts one range per
    frame (modules/cost_volume.py:124-127); the oracle restates that."""
    G = _golden("range", RANGE_CASE)
    oc, ol, op, _ = O.forward_dot(**_range_tuple(), num_depth_bins=RANGE_CASE[4], sampler="aten")
    assert torch.equal(op.contiguous(), G["planes"])
    assert (oc - G["cost"]).abs().max().item() <= 2e-6 * float(G["cost"].abs().max()) and torch.equal(ol, G["lowest"])
