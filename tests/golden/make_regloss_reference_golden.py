"""Writes tests/golden/reference/regloss_oracle_vs_reference.npz: the seeded inputs of
tests/test_regloss_oracle_vs_reference.py and the outputs of the unmodified reference DepthModel.compute_losses
(experiment_modules/depth_model.py) on them, run with the restated kornia filters of oracle/gradloss_oracle.py and
oracle/normals_oracle.py and the stand-ins of oracle/regloss_oracle.py (see tests/refgolden.py).  Only this file is
written.

    SIMPLERECON_REF=<SimpleRecon source tree> python tests/golden/make_regloss_reference_golden.py
"""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from oracle.ref_import import reference_available  # noqa: E402
from tests import refgolden  # noqa: E402

if __name__ == "__main__":
    if not reference_available():
        sys.exit("set $SIMPLERECON_REF to the SimpleRecon source tree")
    from tests import test_regloss_oracle_vs_reference as mod
    out = refgolden.save("regloss_oracle_vs_reference", mod.reference_outputs())
    print(f"{out.relative_to(ROOT)}: {out.stat().st_size} bytes")
