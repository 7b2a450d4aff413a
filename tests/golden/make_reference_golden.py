"""Writes tests/golden/reference/*.npz: the outputs of the unmodified SimpleRecon code for the seeded
inputs of the tests that pin the oracles to it (see tests/refgolden.py).

    SIMPLERECON_REF=<SimpleRecon source tree> python tests/golden/make_reference_golden.py
"""
import importlib
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from oracle.ref_import import reference_available  # noqa: E402
from tests import refgolden  # noqa: E402

MODULES = ("oracle_vs_reference", "tsdf_oracle_vs_reference", "mvs_oracle_vs_reference",
           "mvdepth_oracle_vs_reference", "emu_python_stack", "boundary")

if __name__ == "__main__":
    if not reference_available():
        sys.exit("set $SIMPLERECON_REF to the SimpleRecon source tree")
    for name in MODULES:
        mod = importlib.import_module(f"tests.test_{name}")
        out = refgolden.save(name, mod.reference_outputs())
        print(f"{out.relative_to(ROOT)}: {out.stat().st_size} bytes")
