"""Writes tests/golden/reference/mesh_vs_reference.npz: the outputs of the unmodified SimpleRecon
TSDF mesh export for the seeded inputs of tests/test_mesh_vs_reference.py (see tests/refgolden.py).
Only this file is written; the other stored outputs come from make_reference_golden.py.

    SIMPLERECON_REF=<SimpleRecon source tree> python tests/golden/make_mesh_reference_golden.py
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
    from tests import test_mesh_vs_reference as mod
    out = refgolden.save("mesh_vs_reference", mod.reference_outputs())
    print(f"{out.relative_to(ROOT)}: {out.stat().st_size} bytes")
