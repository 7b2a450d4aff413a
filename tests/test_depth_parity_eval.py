"""CPU half of the depth-map parity check: when a GPU run left scripts/depth_parity.py's DUMP
(tests/test_gpu_depth_parity.py) and the reference tree is mounted, push the reference's and our
cost volumes through the reference's own CVEncoder + DepthDecoderPP (seeded weights) and require
depth Abs-Diff <= 1e-4 on every frame (utils/metrics_utils.py:38; BASELINE.json north_star)."""
import importlib.util
from pathlib import Path

import pytest

from oracle.ref_import import reference_available

ROOT = Path(__file__).resolve().parents[1]


@pytest.mark.skipif(not reference_available(), reason="reference tree not mounted")
def test_depth_abs_diff_through_the_reference_unet():
    spec = importlib.util.spec_from_file_location("depth_parity", ROOT / "scripts" / "depth_parity.py")
    dp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dp)
    if not dp.DUMP.is_file():
        pytest.skip("no GPU dump (run tests/test_gpu_depth_parity.py on the GPU first)")
    import numpy as np
    z = np.load(dp.DUMP)
    if z["hero_cost"].shape[0] != dp.FRAMES["hero"] or z["dot_cost"].shape[0] != dp.FRAMES["dot"]:
        pytest.skip("stale dump of an earlier round (different frame counts)")
    rep = dp.evaluate(write=True)
    for kind in ("dot", "hero"):
        assert rep[kind]["frames"] == dp.FRAMES[kind]
        assert rep[kind]["depth_abs_diff_worst_frame"] <= 1e-4, rep[kind]
        assert rep[kind]["argmax_plane_mismatch_px"] <= 0.005 * rep[kind]["frames"] * 120 * 160
