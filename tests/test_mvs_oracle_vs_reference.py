"""CPU: the multi-view consistency oracle against the unmodified reference process_depth
(tools/torch_point_cloud_fusion.py, its hard-wired .cuda() calls made no-ops when the stored outputs
are generated; stored under tests/golden/reference/, see tests/refgolden.py)."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import mvs_oracle as M
from simplerecon_b200.synthetic import make_mvs_scene
from tests import refgolden

def _load_reference_fuser(monkeypatch):
    from oracle.ref_import import reference_root
    import sys
    import types
    if "tqdm" not in sys.modules:
        try:
            import tqdm  # noqa: F401
        except Exception:
            m = types.ModuleType("tqdm")
            m.tqdm = lambda x, **k: x
            sys.modules["tqdm"] = m
    spec = importlib.util.spec_from_file_location(
        "_simplerecon_ref_pcfusion", os.path.join(reference_root(), "tools", "torch_point_cloud_fusion.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)      # process_depth hard-wires .cuda()
    return mod


CASES = [(1, 5, (24, 32)), (2, 9, (30, 40))]


def _ref_indices(n):
    return (0, n // 2)


def reference_outputs():
    """For tests/golden/make_reference_golden.py."""
    import _pytest.monkeypatch
    mp = _pytest.monkeypatch.MonkeyPatch()
    try:
        R = _load_reference_fuser(mp)
        out = {}
        for seed, n, hw in CASES:
            sc = make_mvs_scene(seed=seed, frames=n, height=hw[0], width=hw[1])
            depths, images, P, K = sc["depths"], sc["images"], sc["cam_T_world"], sc["K"]
            for ref_idx in _ref_indices(n):
                src = torch.arange(n) != ref_idx
                rp, rrgb, rvalid = R.process_depth(depths[ref_idx], images[ref_idx], depths[src], images[src],
                                                   P[ref_idx], P[src], K[ref_idx], K[src], 0.1, 3)
                out[f"{seed}_{n}_{ref_idx}"] = dict(points=np.asarray(rp), rgb=np.asarray(rrgb), valid=np.asarray(rvalid))
        return out
    finally:
        mp.undo()


@pytest.mark.parametrize("seed,n,hw", CASES)
def test_process_depth_matches_live_reference(seed, n, hw):
    sc = make_mvs_scene(seed=seed, frames=n, height=hw[0], width=hw[1])
    depths, images, P, K = sc["depths"], sc["images"], sc["cam_T_world"], sc["K"]
    for ref_idx in _ref_indices(n):
        G = refgolden.load("mvs_oracle_vs_reference", f"{seed}_{n}_{ref_idx}")
        rp, rrgb, rvalid = G["points"].numpy(), G["rgb"].numpy(), G["valid"].numpy()
        src = torch.arange(n) != ref_idx
        pts_avg, n_valid, valid = M.process_depth_dense(depths[ref_idx], depths[src], P[ref_idx], P[src],
                                                        K[ref_idx], K[src], 0.1, 3)
        assert np.array_equal(valid.numpy(), rvalid) and 0.05 < valid.float().mean().item() < 0.99
        op, orgb = M.compact(pts_avg, valid, images[ref_idx])
        assert np.allclose(op.numpy(), rp, rtol=0, atol=1e-6) and np.array_equal(orgb.numpy(), rrgb)
