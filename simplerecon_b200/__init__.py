"""simplerecon_b200 — H100-native plane-sweep cost volume behind SimpleRecon's
``CostVolumeManager`` / ``FeatureVolumeManager`` API.

Only the hot path named by BASELINE.json is here: the cost-volume build of the
reference's ``modules/cost_volume.py``, as hand-written sm_90a kernels in
``csrc/`` behind a C ABI (``include/srcv_b200.h``), plus the Python mirror of the
reference's manager classes that binds it.  Encoders, decoder, datasets and
training stay the reference's own PyTorch code.
"""
from .cost_volume import (CostVolumeManager, FastFeatureVolumeManager, FeatureVolumeManager,
                          instance_norm_to_chunk_planar)
from .geometry import BackprojectDepth, Project3D, pose_distance
from .install import install, uninstall
from .networks import MLP
from . import torch_ops  # noqa: E402,F401  registers torch.ops.b200cv.{dot_forward,dot_backward,mlp_forward}

__all__ = [
    "CostVolumeManager", "FeatureVolumeManager", "FastFeatureVolumeManager", "MLP",
    "BackprojectDepth", "Project3D", "pose_distance", "install", "uninstall",
]
__version__ = "0.1.0"
from .tsdf import TSDF, TSDFFuser  # noqa: E402,F401  (reference tools/tsdf.py)
from .fusers import ColorFuser  # noqa: E402,F401  (OurFuser with colour, DESIGN §4.11)
from . import point_cloud_fusion  # noqa: E402,F401  (reference tools/torch_point_cloud_fusion.py)
from .losses import MSGradientLoss, MVDepthLoss, ScaleInvariantLoss  # noqa: E402,F401  (reference losses.py:11-54, :79-208)
from .losses import depth_regression_losses  # noqa: E402,F401  (reference experiment_modules/depth_model.py:447-474)
from .metrics import compute_depth_metrics, compute_depth_metrics_batched, depth_metrics  # noqa: E402,F401  (reference utils/metrics_utils.py)
from .normals import NormalGenerator, NormalsLoss  # noqa: E402,F401  (reference geometry_utils.py:92-133, losses.py:57-77)
