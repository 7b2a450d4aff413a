"""Swap the fused managers into a SimpleRecon checkout.

``install()`` replaces ``CostVolumeManager``, ``FeatureVolumeManager`` and
``FastFeatureVolumeManager`` in the reference's ``modules.cost_volume`` namespace
(and in ``experiment_modules.depth_model`` if it was already imported, because it
binds the names at import time — reference experiment_modules/depth_model.py:10-11)
so ``DepthModel`` builds the sm_90a-backed classes without any edit to the
reference.  ``install(losses=True)`` also swaps the reference's ``losses.MVDepthLoss`` (the
training loss of depth_model.py:144, :477-485) for the kernel-backed mirror.  ``install(fusion=True)``
swaps ``tools.tsdf.TSDF`` / ``TSDFFuser`` for the kernel-backed mirrors (fusion and mesh export), and
the names ``tools.fusers_helper`` bound at import (tools/fusers_helper.py:8) if it was already
imported.  ``install(fusion=True, fuse_color=True)`` also wraps ``tools.fusers_helper.get_fuser`` so that
``--depth_fuser ours --fuse_color`` gets a ``fusers.ColorFuser`` (colour fused on the GPU) instead of the
reference's warning and a colourless ``OurFuser``; every other option goes to the original.
``install(metrics=True)`` swaps ``compute_depth_metrics`` / ``compute_depth_metrics_batched`` of
``utils.metrics_utils`` (and the name ``experiment_modules.depth_model`` binds at import, :16, if it was
already imported) for wrappers that run CUDA tensors through the metrics kernel and hand anything else to
the saved originals, so CPU callers of that utility module keep working.
``install(normals=True)`` swaps ``utils.geometry_utils.NormalGenerator`` and ``losses.NormalsLoss`` (the
normals term of the training loss, depth_model.py:143, :156, :475) for the kernel-backed mirrors, and the
names ``experiment_modules.depth_model`` binds at import (:7, :15) if it was already imported.
``install(depth_losses=True)`` swaps ``losses.MSGradientLoss`` and ``losses.ScaleInvariantLoss`` (the gradient
term of the training loss and the logged scale-invariant term, depth_model.py:466-468, :487) for the
kernel-backed mirrors, and the names ``experiment_modules.depth_model`` binds at import (:7) if it was already
imported.
``install(regression_losses=True)`` imports ``experiment_modules.depth_model`` and replaces
``DepthModel.compute_losses`` (:409-500) with ``losses.compute_losses``: the multi-scale log-L1 loss and the logged
regression terms from one fused call, the other terms from the model's own loss modules.  Models whose multi-scale
loss is not the mean ``nn.L1Loss``, and CPU ground truth, go to the saved original.  With this flag the other flags
also patch ``experiment_modules.depth_model``, since it is imported first.
``uninstall()`` restores everything.  See INTEGRATION.md.
"""
from __future__ import annotations

import importlib
import sys

import torch

_NAMES = ("CostVolumeManager", "FeatureVolumeManager", "FastFeatureVolumeManager")
_saved: dict = {}


def install(verbose: bool = False, losses: bool = False, fusion: bool = False, fuse_color: bool = False,
            metrics: bool = False, normals: bool = False, depth_losses: bool = False,
            regression_losses: bool = False) -> list[str]:
    """Returns the list of patched module names.  Requires the reference checkout to
    be importable (on ``sys.path``) as ``modules.cost_volume``; with ``losses=True`` also as ``losses``,
    with ``fusion=True`` also as ``tools.tsdf``, with ``fuse_color=True`` also as ``tools.fusers_helper``,
    with ``metrics=True`` also as ``utils.metrics_utils``, with ``normals=True`` also as ``losses`` and
    ``utils.geometry_utils``, with ``depth_losses=True`` also as ``losses``, with ``regression_losses=True``
    also as ``experiment_modules.depth_model``."""
    if fuse_color and not fusion:
        raise ValueError("install(fuse_color=True) needs fusion=True: colour is fused into the kernel-backed TSDF")
    from . import cost_volume as ours
    patched = []
    ref_cv = importlib.import_module("modules.cost_volume")
    targets = [ref_cv]
    if regression_losses:
        importlib.import_module("experiment_modules.depth_model")
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
    if fusion:
        from . import tsdf as ours_tsdf
        ref_tsdf = importlib.import_module("tools.tsdf")
        fh = importlib.import_module("tools.fusers_helper") if fuse_color else sys.modules.get("tools.fusers_helper")
        for mod in [ref_tsdf] + ([fh] if fh is not None else []):
            for n in ("TSDF", "TSDFFuser"):
                if hasattr(mod, n):
                    _saved.setdefault((mod.__name__, n), getattr(mod, n))
                    setattr(mod, n, getattr(ours_tsdf, n))
            if mod.__name__ not in patched:
                patched.append(mod.__name__)
        if fuse_color:
            _saved.setdefault((fh.__name__, "get_fuser"), fh.get_fuser)
            fh.get_fuser = _color_get_fuser(_saved[(fh.__name__, "get_fuser")], fh)
    if metrics:
        from . import metrics as ours_metrics
        mu = importlib.import_module("utils.metrics_utils")
        for mod in [mu] + ([dm] if dm is not None else []):       # depth_model binds compute_depth_metrics (:16)
            for n in ("compute_depth_metrics", "compute_depth_metrics_batched"):
                if hasattr(mod, n):
                    _saved.setdefault((mod.__name__, n), getattr(mod, n))
                    setattr(mod, n, _cuda_or_original(getattr(ours_metrics, n), _saved[(mod.__name__, n)]))
            if mod.__name__ not in patched:
                patched.append(mod.__name__)
    if normals:
        from . import normals as ours_normals
        for mod_name, n in (("utils.geometry_utils", "NormalGenerator"), ("losses", "NormalsLoss")):
            for mod in [importlib.import_module(mod_name)] + ([dm] if dm is not None else []):
                if hasattr(mod, n):
                    _saved.setdefault((mod.__name__, n), getattr(mod, n))
                    setattr(mod, n, getattr(ours_normals, n))
                    if mod.__name__ not in patched:
                        patched.append(mod.__name__)
    if depth_losses:
        from . import losses as ours_losses
        for mod in [importlib.import_module("losses")] + ([dm] if dm is not None else []):
            for n in ("MSGradientLoss", "ScaleInvariantLoss"):
                if hasattr(mod, n):
                    _saved.setdefault((mod.__name__, n), getattr(mod, n))
                    setattr(mod, n, getattr(ours_losses, n))
            if mod.__name__ not in patched:
                patched.append(mod.__name__)
    if regression_losses:
        from .losses import compute_losses
        _saved.setdefault((dm.__name__, "DepthModel.compute_losses"), dm.DepthModel.compute_losses)
        dm.DepthModel.compute_losses = compute_losses
        if dm.__name__ not in patched:
            patched.append(dm.__name__)
    if verbose:
        print(f"simplerecon_b200: installed fused cost-volume managers into {patched}")
    return patched


def _color_get_fuser(original, fh):
    """``get_fuser`` (tools/fusers_helper.py:188-220) with ``ours`` + ``fuse_color`` -> ``ColorFuser``."""
    def get_fuser(opts, scan):
        if getattr(opts, "depth_fuser", None) != "ours" or not getattr(opts, "fuse_color", False):
            return original(opts, scan)
        from .fusers import ColorFuser
        if opts.dataset == "scannet":      # the ground-truth mesh path exactly as get_fuser computes it
            gt_path = fh.ScannetDataset.get_gt_mesh_path(opts.dataset_path, opts.split, scan)
        else:
            gt_path = None
        return ColorFuser(gt_path=gt_path, fusion_resolution=opts.fusion_resolution,
                          max_fusion_depth=opts.fusion_max_depth, fuse_color=True)
    get_fuser.__wrapped__ = original
    return get_fuser


def _cuda_or_original(fast, original):
    """``fast`` for CUDA ground truth, ``original`` for anything else (CPU callers of the utility module)."""
    def metrics_fn(gt, *args, **kwargs):
        if torch.is_tensor(gt) and gt.is_cuda:
            return fast(gt, *args, **kwargs)
        return original(gt, *args, **kwargs)
    metrics_fn.__name__ = original.__name__
    metrics_fn.__doc__ = fast.__doc__
    metrics_fn.__wrapped__ = original
    return metrics_fn


def saved_original(mod_name: str, name: str):
    """What ``install`` replaced under ``name`` (``Class.attr`` for a class attribute) in module ``mod_name``."""
    try:
        return _saved[(mod_name, name)]
    except KeyError:
        raise RuntimeError(f"{mod_name}.{name} has not been replaced by install(): no original to call") from None


def uninstall() -> None:
    for (mod_name, n), cls in list(_saved.items()):
        mod = sys.modules.get(mod_name)
        if mod is not None:
            *owner, attr = n.split(".")              # "Class.attr" names a class attribute
            for o in owner:
                mod = getattr(mod, o)
            setattr(mod, attr, cls)
    _saved.clear()
