"""Swap the fused managers into a SimpleRecon checkout.

``install()`` replaces ``CostVolumeManager``, ``FeatureVolumeManager`` and
``FastFeatureVolumeManager`` in the reference's ``modules.cost_volume`` namespace
(and in ``experiment_modules.depth_model`` if it was already imported, because it
binds the names at import time — reference experiment_modules/depth_model.py:10-11)
so ``DepthModel`` builds the sm_90a-backed classes without any edit to the
reference.  ``install(losses=True)`` also swaps the reference's ``losses.MVDepthLoss`` (the
training loss of depth_model.py:144, :477-485) for the kernel-backed mirror.  See INTEGRATION.md.
"""
from __future__ import annotations

import importlib
import sys

_NAMES = ("CostVolumeManager", "FeatureVolumeManager", "FastFeatureVolumeManager")
_saved: dict = {}


def install(verbose: bool = False, losses: bool = False) -> list[str]:
    """Returns the list of patched module names.  Requires the reference checkout to
    be importable (on ``sys.path``) as ``modules.cost_volume``; with ``losses=True`` also as ``losses``."""
    from . import cost_volume as ours
    patched = []
    ref_cv = importlib.import_module("modules.cost_volume")
    targets = [ref_cv]
    dm = sys.modules.get("experiment_modules.depth_model")
    if dm is not None:
        targets.append(dm)
    for mod in targets:
        for n in _NAMES:
            if hasattr(mod, n):
                _saved.setdefault((mod.__name__, n), getattr(mod, n))
                setattr(mod, n, getattr(ours, n))
        patched.append(mod.__name__)
    if losses:
        from .losses import MVDepthLoss
        ref_losses = importlib.import_module("losses")
        for mod in [ref_losses] + ([dm] if dm is not None else []):   # depth_model binds the name at import (:7)
            if hasattr(mod, "MVDepthLoss"):
                _saved.setdefault((mod.__name__, "MVDepthLoss"), mod.MVDepthLoss)
                mod.MVDepthLoss = MVDepthLoss
                if mod.__name__ not in patched:
                    patched.append(mod.__name__)
    if verbose:
        print(f"simplerecon_b200: installed fused cost-volume managers into {patched}")
    return patched


def uninstall() -> None:
    for (mod_name, n), cls in list(_saved.items()):
        mod = sys.modules.get(mod_name)
        if mod is not None:
            setattr(mod, n, cls)
    _saved.clear()
