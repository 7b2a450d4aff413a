"""``ColorFuser``: the reference's ``OurFuser`` (tools/fusers_helper.py:22-82) with colour.

The reference fuses colour only through ``Open3DFuser`` (needs open3d, batch 1, a host copy and a CPU
integration per frame); with its default ``ours`` fuser, ``--fuse_color`` prints a warning and drops the
colour (:197-207).  ``ColorFuser`` has ``OurFuser``'s interface and bounds logic and fuses the frames'
colour into the kernel-backed volume (DESIGN §4.11); ``export_mesh`` writes a vertex-coloured binary PLY
without trimesh.  ``install(fusion=True, fuse_color=True)`` makes ``get_fuser`` return it for
``--depth_fuser ours --fuse_color``.  With ``unbounded=True`` and no ground-truth mesh its volume is a
``SparseTSDF`` on the ±10 m cube's lattice instead of that cube (DESIGN §4.16), with or without colour;
``install(fusion=True, unbounded_fusion=True)`` makes ``get_fuser`` use that for ``--depth_fuser ours``.
"""
from __future__ import annotations

from .tsdf import DEFAULT_BOUNDS, SparseTSDF, TSDF, TSDFFuser, colors_to_u8, write_ply


class ColorFuser:
    """OurFuser's constructor, ``fuse_frames``, ``export_mesh`` and ``get_mesh``, with colour."""

    def __init__(self, gt_path="", fusion_resolution=0.04, max_fusion_depth=3, fuse_color=True, unbounded=False,
                 max_blocks=1 << 17):
        self.fusion_resolution = fusion_resolution
        self.max_fusion_depth = max_fusion_depth
        self.fuse_color = bool(fuse_color)
        if gt_path is not None:             # OurFuser's bounds: the ground-truth mesh's extent (:48-50)
            import trimesh
            gt_mesh = trimesh.load(gt_path, force="mesh")
            tsdf_pred = TSDF.from_mesh(gt_mesh, voxel_size=fusion_resolution, color=self.fuse_color)
        elif unbounded:                     # no bounds: voxel blocks where the frames reach, on the cube's lattice
            tsdf_pred = SparseTSDF(fusion_resolution, max_blocks=max_blocks, color=self.fuse_color)
        else:                               # or a ±10 m cube (:51-60)
            tsdf_pred = TSDF.from_bounds(dict(DEFAULT_BOUNDS), voxel_size=fusion_resolution, color=self.fuse_color)
        self.tsdf_fuser_pred = TSDFFuser(tsdf_pred, max_depth=max_fusion_depth)

    def fuse_frames(self, depths_b1hw, K_b44, cam_T_world_b44, color_b3hw):
        """Depth, K and pose go in as ``.half()`` as in OurFuser (:64-71); ``color_b3hw`` is the
        dataloader's ImageNet-normalised image at any resolution (ignored when ``fuse_color`` is False)."""
        self.tsdf_fuser_pred.integrate_depth(
            depth_b1hw=depths_b1hw.half(),
            cam_T_world_T_b44=cam_T_world_b44.half(),
            K_b44=K_b44.half(),
            color_b3hw=color_b3hw if self.fuse_color else None,
        )

    def export_mesh(self, path, export_single_mesh=True):
        """Binary PLY at ``path`` (vertex colours when fusing colour); needs no trimesh."""
        tsdf = self.tsdf_fuser_pred.tsdf
        if self.fuse_color:
            verts, faces, _, colors = tsdf.extract_mesh(single_mesh=export_single_mesh, with_colors=True)
            write_ply(path, verts.cpu().numpy(), faces.cpu().numpy(), colors_to_u8(colors))
        else:
            verts, faces, _ = tsdf.extract_mesh(single_mesh=export_single_mesh)
            write_ply(path, verts.cpu().numpy(), faces.cpu().numpy())

    def get_mesh(self, export_single_mesh=True, convert_to_trimesh=True):
        """A ``trimesh.Trimesh`` with ``vertex_colors`` (as OurFuser, ``convert_to_trimesh`` is ignored)."""
        return self.tsdf_fuser_pred.tsdf.to_mesh(export_single_mesh=export_single_mesh)
