"""GPU half of the depth-map parity check (BASELINE target: depth Abs-Diff <= 1e-4 through the
reference's U-Net): our cost volumes for a batch of seeded 640x480 tuples — 8 hero frames in one
B = 8 call, 4 dot frames — written to scripts/depth_parity.py's DUMP.  The reference's decoder
exists only in the SimpleRecon source tree, so the evaluation is tests/test_depth_parity_eval.py there
(scripts/depth_parity.py holds both halves)."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def test_dump_cost_volumes_for_depth_parity(cuda_device):
    spec = importlib.util.spec_from_file_location("depth_parity", ROOT / "scripts" / "depth_parity.py")
    dp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dp)
    dp.dump()
    z = np.load(dp.DUMP)
    assert z["hero_cost"].shape == (8, 64, 120, 160) and z["dot_cost"].shape == (4, 64, 120, 160)
    assert np.isfinite(z["hero_cost"]).all() and np.isfinite(z["dot_cost"]).all()
    assert "wgmma" in str(z["hero_variant"]) and "fast" in str(z["dot_variant"])
