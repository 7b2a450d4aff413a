"""Writes tests/golden/reference/metrics_oracle_vs_reference.npz: the seeded edge-case inputs of
tests/test_metrics_oracle_vs_reference.py and the outputs of the unmodified reference
utils/metrics_utils.py on them (see tests/refgolden.py).  Only this file is written.

    SIMPLERECON_REF=<SimpleRecon source tree> python tests/golden/make_metrics_reference_golden.py
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
    from tests import test_metrics_oracle_vs_reference as mod
    out = refgolden.save("metrics_oracle_vs_reference", mod.reference_outputs())
    print(f"{out.relative_to(ROOT)}: {out.stat().st_size} bytes")
