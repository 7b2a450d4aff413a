"""Import the UNMODIFIED reference classes from the SimpleRecon source tree named by
``$SIMPLERECON_REF``.

TEST INFRASTRUCTURE — never imported by the product package.

The tests never need the reference tree: this module is used by the scripts under
``tests/golden/`` that generate the committed golden vectors and stored reference outputs,
and by the two tests of ``install()`` against the real reference modules, which skip
without it.

Why stubs: ``modules/cost_volume.py`` itself needs only torch + einops, but its
imports pull ``modules/networks.py:1,4`` (antialiased_cnns, timm),
``utils/generic_utils.py:6`` and ``utils/geometry_utils.py:1`` (kornia), none of
which is installed in this image, and ``utils/generic_utils.py:87-94`` compiles a
TorchScript function that names ``kornia.filters.blur_pool2d`` at import time.
We register inert stand-ins for those four packages; nothing on the cost-volume
path ever calls into them.  TorchScript stays ON, so ``BackprojectDepth`` and
``Project3D`` run as the real ``ScriptModule``s they are in the reference.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

REF_ENV = "SIMPLERECON_REF"


def reference_root() -> str | None:
    c = os.environ.get(REF_ENV)
    if c and os.path.isfile(os.path.join(c, "modules", "cost_volume.py")):
        return c
    return None


def reference_available() -> bool:
    return reference_root() is not None


def _install_stubs() -> None:
    import torch

    if "kornia" not in sys.modules:
        kornia = types.ModuleType("kornia")
        filters = types.ModuleType("kornia.filters")

        def blur_pool2d(x: torch.Tensor, kernel_size: int) -> torch.Tensor:
            # never executed on the cost-volume path; present so that
            # utils/generic_utils.py:87-94 (pyrdown) can be TorchScript-compiled.
            return torch.nn.functional.avg_pool2d(x, 2)

        filters.blur_pool2d = blur_pool2d
        kornia.filters = filters
        sys.modules["kornia"] = kornia
        sys.modules["kornia.filters"] = filters
    for name in ("timm", "antialiased_cnns"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)


_cached = None


def load_reference():
    """Returns a namespace with the reference's cost-volume classes and helpers."""
    global _cached
    if _cached is not None:
        return _cached
    root = reference_root()
    if root is None:
        raise RuntimeError(
            "reference tree not found (set $SIMPLERECON_REF to the SimpleRecon source tree)"
        )
    _install_stubs()
    if root not in sys.path:
        sys.path.insert(0, root)
    # The reference's top-level packages are called `modules` and `utils`; make
    # sure nothing else with those names is shadowing them.
    for top in ("modules", "utils"):
        m = sys.modules.get(top)
        if m is not None and not getattr(m, "__file__", "").startswith(root) \
                and not any(str(p).startswith(root) for p in getattr(m, "__path__", [])):
            del sys.modules[top]
    cv = importlib.import_module("modules.cost_volume")
    nets = importlib.import_module("modules.networks")
    geo = importlib.import_module("utils.geometry_utils")
    ns = types.SimpleNamespace(
        root=root,
        cost_volume=cv,
        networks=nets,
        geometry=geo,
        CostVolumeManager=cv.CostVolumeManager,
        FeatureVolumeManager=cv.FeatureVolumeManager,
        FastFeatureVolumeManager=cv.FastFeatureVolumeManager,
        MLP=nets.MLP,
        CVEncoder=nets.CVEncoder,
        DepthDecoderPP=nets.DepthDecoderPP,
        BackprojectDepth=geo.BackprojectDepth,
        Project3D=geo.Project3D,
        pose_distance=geo.pose_distance,
    )
    _cached = ns
    return ns


_cached_tsdf = None


def load_reference_tsdf():
    """The reference's ``tools/tsdf.py`` (``TSDF``, ``TSDFFuser``) imported unmodified.  It
    imports trimesh and skimage at module level (mesh export / marching cubes, not on the
    integration path); neither is installed here, so inert stand-ins are registered."""
    global _cached_tsdf
    if _cached_tsdf is not None:
        return _cached_tsdf
    root = reference_root()
    if root is None:
        raise RuntimeError("reference tree not found (set $SIMPLERECON_REF to the SimpleRecon source tree)")
    for name in ("trimesh", "skimage", "skimage.measure"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["skimage"].measure = sys.modules["skimage.measure"]
    if not hasattr(sys.modules["trimesh"], "Trimesh"):
        sys.modules["trimesh"].Trimesh = object
    import importlib.util
    spec = importlib.util.spec_from_file_location("_simplerecon_ref_tsdf", os.path.join(root, "tools", "tsdf.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    _cached_tsdf = types.SimpleNamespace(TSDF=mod.TSDF, TSDFFuser=mod.TSDFFuser, module=mod)
    return _cached_tsdf
