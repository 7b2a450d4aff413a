"""Stored outputs of the unmodified SimpleRecon code for the tests that pin the oracles to it: each
such module's ``reference_outputs()`` runs the original on its seeded inputs, and
``tests/golden/make_reference_golden.py`` (needs ``$SIMPLERECON_REF``) saves them under
``tests/golden/reference/``, so the tests run anywhere."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import torch

GOLDEN_DIR = Path(__file__).resolve().parent / "golden" / "reference"


def save(module: str, cases: dict) -> Path:
    """cases = {case: {name: tensor | float}} -> GOLDEN_DIR/<module>.npz with keys "<case>/<name>"."""
    GOLDEN_DIR.mkdir(parents=True, exist_ok=True)
    flat = {}
    for case, arrays in cases.items():
        for name, v in arrays.items():
            flat[f"{case}/{name}"] = v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)
    out = GOLDEN_DIR / f"{module}.npz"
    np.savez_compressed(out, **flat)
    return out


_cache: dict[str, dict] = {}


def load(module: str, case: str) -> dict[str, torch.Tensor]:
    """{name: tensor} of one stored case (arrays of strings stay numpy arrays)."""
    if module not in _cache:
        with np.load(GOLDEN_DIR / f"{module}.npz") as z:
            _cache[module] = {k: z[k] for k in z.files}
    prefix = f"{case}/"
    return {k[len(prefix):]: torch.from_numpy(v.copy()) if v.dtype.kind in "biuf" else v
            for k, v in _cache[module].items() if k.startswith(prefix)}
