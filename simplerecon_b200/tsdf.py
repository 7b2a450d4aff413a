"""Dense-grid TSDF fusion of predicted depth maps and mesh extraction, backed by sm_90a kernels.

Mirrors the reference's ``tools/tsdf.py`` — ``TSDF`` (:11-170, the volume, its bounds arithmetic and
mesh export) and ``TSDFFuser`` (:173-320, ``integrate_depth``) — as ``OurFuser`` uses them
(``tools/fusers_helper.py:22-82``): same constructor / method names, argument meaning and fp16
state, so ``test.py`` can fuse and export meshes through these classes unchanged.

Mesh extraction (``extract_mesh``, and ``to_mesh`` / ``save`` on top of it) is a marching-cubes
kernel (csrc/srcv_mesh.cuh) whose output is defined in DESIGN §4.10 rather than byte-matched to
scikit-image: one canonically ordered vertex per crossing edge, a generated triangulation table that
keeps the surface closed and oriented toward free space, no degenerate triangles.
``export_single_mesh=True`` is read as: only cubes whose 8 corners all carry weight are meshed
(the reference needs a custom scikit-image fork for that flag; this is our definition of it).

Differences, by design: ``voxel_coords`` is not stored (the kernel recomputes the 6 bytes per
voxel from the grid index; the property materialises it on demand), a batch of frames is ONE
launch (frames are applied in order inside the kernel), ``save`` writes the PLY itself without
moving the volume to the CPU (the reference's ``save`` calls ``self.cpu()`` first), and there is
no CPU path: CUDA tensors on an sm_90 device, or an exception.

Colour (DESIGN §4.11, this library's definition: the reference's ``OurFuser`` has none): a volume made
with ``color=True`` carries an fp32 (3,X,Y,Z) ``tsdf_colors`` volume, ``integrate_depth`` then takes
``color_b3hw`` and averages it in with the values' own weights (values and weights stay bit-identical to
the plain path), and ``extract_mesh`` / ``to_mesh`` / ``save`` produce vertex colours.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Tuple

import numpy as np
import torch

from . import _native


class TSDF:
    """Volume container (reference tools/tsdf.py:11-130)."""

    VOX_MOD = 8   # final voxel volume dimensions are multiples of 8 (:17)

    def __init__(self, tsdf_values: torch.Tensor, tsdf_weights: torch.Tensor, voxel_size: float,
                 origin: torch.Tensor, colors: torch.Tensor | None = None):
        self.tsdf_values = tsdf_values.half().contiguous()
        self.tsdf_weights = tsdf_weights.half().contiguous()
        self.voxel_size = float(voxel_size)
        self.origin = origin.float()          # kept in fp32: the coordinates are built in fp32 and then halved (:99-110, :92)
        self.tsdf_colors = None               # (3,X,Y,Z) fp32 R, G, B in [0, 1], or None (DESIGN §4.11)
        if colors is not None:
            if tuple(colors.shape) != (3, *self.tsdf_values.shape):
                raise ValueError(f"colors must be (3, X, Y, Z) = (3, {', '.join(map(str, self.tsdf_values.shape))}), "
                                 f"got {tuple(colors.shape)}")
            self.tsdf_colors = colors.float().contiguous()

    @classmethod
    def from_bounds(cls, bounds: dict, voxel_size: float, device="cuda", color: bool = False):
        """-1 / 0 initialised volume covering ``bounds`` (:70-97); ``color=True`` adds a 0-initialised
        colour volume (12 bytes per voxel)."""
        for key in ("xmin", "xmax", "ymin", "ymax", "zmin", "zmax"):
            if key not in bounds:
                raise KeyError("Provided bounds dict need to have keys 'xmin', 'xmax', 'ymin', 'ymax', 'zmin', 'zmax'!")
        dims = tuple(int(np.ceil((bounds[a + "max"] - bounds[a + "min"]) / voxel_size / cls.VOX_MOD)) * cls.VOX_MOD
                     for a in "xyz")
        origin = torch.tensor([bounds["xmin"], bounds["ymin"], bounds["zmin"]], dtype=torch.float32)
        values = -torch.ones(dims, dtype=torch.float16, device=device)
        weights = torch.zeros(dims, dtype=torch.float16, device=device)
        colors = torch.zeros((3, *dims), dtype=torch.float32, device=device) if color else None
        return cls(values, weights, voxel_size, origin, colors)

    @classmethod
    def generate_voxel_coords(cls, origin: torch.Tensor, volume_dims: Tuple[int, int, int], voxel_size: float):
        """World coordinates of every voxel, (3,X,Y,Z) (:99-110)."""
        grid = torch.meshgrid([torch.arange(vd, device=origin.device) for vd in volume_dims], indexing="ij")
        return origin.view(3, 1, 1, 1) + torch.stack(grid, 0) * voxel_size

    @property
    def voxel_coords(self) -> torch.Tensor:
        """fp16 (3,X,Y,Z), materialised on demand (the kernel does not read it)."""
        return self.generate_voxel_coords(self.origin.to(self.tsdf_values.device), tuple(self.tsdf_values.shape),
                                          self.voxel_size).half()

    @classmethod
    def from_mesh(cls, mesh, voxel_size: float, device="cuda", color: bool = False):
        """Volume covering ``mesh.vertices`` plus 3 voxels on every side (:51-67)."""
        verts = np.asarray(mesh.vertices)
        xmax, ymax, zmax = verts.max(0)
        xmin, ymin, zmin = verts.min(0)
        bounds = {"xmin": xmin, "xmax": xmax, "ymin": ymin, "ymax": ymax, "zmin": zmin, "zmax": zmax}
        for key, val in bounds.items():
            bounds[key] = val - 3 * voxel_size if "min" in key else val + 3 * voxel_size
        return cls.from_bounds(bounds, voxel_size, device=device, color=color)

    @torch.no_grad()
    def extract_mesh(self, scale_to_world: bool = True, single_mesh: bool = False, with_colors: bool = False):
        """Marching cubes at level 0 on the GPU (DESIGN §4.10).  Returns ``(verts (V,3) float32,
        faces (F,3) int32, normals (V,3) float32)`` on the volume's device; one host synchronisation
        (the vertex / face counts).  World coordinates use the origin rounded to fp16, as the
        reference's half ``origin`` does (:34, :154).  ``with_colors=True`` (a colour volume only) appends
        the vertex colours, (V,3) float32 in [0, 1] (DESIGN §4.11); the other three are unchanged."""
        if with_colors and self.tsdf_colors is None:
            raise ValueError("with_colors=True needs a colour volume (TSDF.from_bounds(..., color=True))")
        values, weights = self.tsdf_values, self.tsdf_weights
        _require_cuda(values)
        dev = values.device
        lib = _native.load()
        a = _native.MeshArgs()
        a.tsdf_values, a.tsdf_weights = values.data_ptr(), weights.data_ptr()
        a.X, a.Y, a.Z = (int(d) for d in values.shape)
        origin_h = self.origin.detach().cpu().half().float()
        for i in range(3):
            a.origin[i] = float(origin_h[i])
        a.voxel_size, a.scale_to_world, a.single_mesh = self.voxel_size, int(bool(scale_to_world)), int(bool(single_mesh))
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            n = lib.srcv_mesh_workspace_bytes(C.byref(a))
            ws = torch.empty(n, device=dev, dtype=torch.uint8)
            counts = torch.empty(2, device=dev, dtype=torch.int64)
            _native.check(lib.srcv_mesh_count(C.byref(a), C.c_void_p(counts.data_ptr()), C.c_void_p(ws.data_ptr()), n,
                                              stream))
            V, F = (int(c) for c in counts.tolist())
            verts = torch.empty((V, 3), device=dev, dtype=torch.float32)
            normals = torch.empty((V, 3), device=dev, dtype=torch.float32)
            faces = torch.empty((F, 3), device=dev, dtype=torch.int32)
            if with_colors:
                colors = torch.empty((V, 3), device=dev, dtype=torch.float32)
                _native.check(lib.srcv_mesh_extract_color(
                    C.byref(a), C.c_void_p(self.tsdf_colors.data_ptr()), C.c_void_p(verts.data_ptr() if V else 0),
                    C.c_void_p(normals.data_ptr() if V else 0), C.c_void_p(colors.data_ptr() if V else 0),
                    C.c_void_p(faces.data_ptr() if F else 0), V, F, C.c_void_p(ws.data_ptr()), n, stream))
                return verts, faces, normals, colors
            _native.check(lib.srcv_mesh_extract(C.byref(a), C.c_void_p(verts.data_ptr() if V else 0),
                                                C.c_void_p(normals.data_ptr() if V else 0),
                                                C.c_void_p(faces.data_ptr() if F else 0), V, F,
                                                C.c_void_p(ws.data_ptr()), n, stream))
        return verts, faces, normals

    def to_mesh(self, scale_to_world: bool = True, export_single_mesh: bool = False):
        """A ``trimesh.Trimesh`` built as the reference builds it (:156).  Needs trimesh; without
        it, use ``extract_mesh`` (tensors) or ``save`` (PLY file)."""
        try:
            import trimesh
        except ImportError as e:
            raise ImportError("TSDF.to_mesh needs trimesh; TSDF.extract_mesh returns the mesh as tensors and "
                              "TSDF.save writes a PLY file without it") from e
        if self.tsdf_colors is not None:     # vertex colours as uint8 rint(255 c) (DESIGN §4.11)
            verts, faces, norms, colors = self.extract_mesh(scale_to_world=scale_to_world,
                                                            single_mesh=export_single_mesh, with_colors=True)
            return trimesh.Trimesh(vertices=verts.cpu().numpy(), faces=faces.cpu().numpy(),
                                   normals=norms.cpu().numpy(), vertex_colors=colors_to_u8(colors))
        verts, faces, norms = self.extract_mesh(scale_to_world=scale_to_world, single_mesh=export_single_mesh)
        return trimesh.Trimesh(vertices=verts.cpu().numpy(), faces=faces.cpu().numpy(), normals=norms.cpu().numpy())

    def save(self, savepath, filename, save_mesh: bool = True):
        """Writes the mesh to ``savepath/filename`` with ``.bin`` replaced by ``.ply`` (:159-168):
        binary little-endian PLY, float x/y/z vertices, uchar-counted int faces.  Unlike the
        reference this does not move the volume to the CPU, and it needs no trimesh.  A colour volume
        adds uchar red / green / blue vertex properties."""
        os.makedirs(savepath, exist_ok=True)
        if save_mesh:
            path = os.path.join(savepath, filename).replace(".bin", ".ply")
            if self.tsdf_colors is not None:
                verts, faces, _, colors = self.extract_mesh(with_colors=True)
                write_ply(path, verts.cpu().numpy(), faces.cpu().numpy(), colors_to_u8(colors))
            else:
                verts, faces, _ = self.extract_mesh()
                write_ply(path, verts.cpu().numpy(), faces.cpu().numpy())

    def cuda(self):
        self.tsdf_values = self.tsdf_values.cuda()
        self.tsdf_weights = self.tsdf_weights.cuda()
        if self.tsdf_colors is not None:
            self.tsdf_colors = self.tsdf_colors.cuda()
        return self

    def cpu(self):
        self.tsdf_values = self.tsdf_values.cpu()
        self.tsdf_weights = self.tsdf_weights.cpu()
        if self.tsdf_colors is not None:
            self.tsdf_colors = self.tsdf_colors.cpu()
        return self


def colors_to_u8(colors) -> np.ndarray:
    """(V,3) colours in [0, 1] -> uint8 rint(255 c) (round half to even), as a host array."""
    c = colors.detach().cpu().numpy() if torch.is_tensor(colors) else np.asarray(colors)
    return np.rint(np.float32(255.0) * np.clip(c.astype(np.float32), 0.0, 1.0)).astype(np.uint8)


def write_ply(path, verts: np.ndarray, faces: np.ndarray, colors: np.ndarray | None = None) -> None:
    """Binary little-endian PLY: float x, y, z (and uchar red, green, blue when ``colors`` is given:
    uint8 as is, floats in [0, 1] through ``colors_to_u8``) per vertex; a uchar count and int indices per
    face."""
    verts = np.ascontiguousarray(verts, dtype="<f4").reshape(-1, 3)
    faces = np.ascontiguousarray(faces, dtype="<i4").reshape(-1, 3)
    vprops = "property float x\nproperty float y\nproperty float z\n"
    if colors is not None:
        colors = np.asarray(colors)
        colors = (colors if colors.dtype == np.uint8 else colors_to_u8(colors)).reshape(-1, 3)
        if len(colors) != len(verts):
            raise ValueError(f"{len(colors)} colours for {len(verts)} vertices")
        vprops += "property uchar red\nproperty uchar green\nproperty uchar blue\n"
        vrec = np.empty(len(verts), dtype=[("p", "<f4", (3,)), ("c", "u1", (3,))])
        vrec["p"], vrec["c"] = verts, colors
        vbytes = vrec.tobytes()
    else:
        vbytes = verts.tobytes()
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(verts)}\n{vprops}"
              f"element face {len(faces)}\nproperty list uchar int vertex_indices\nend_header\n")
    rec = np.empty(len(faces), dtype=[("n", "u1"), ("v", "<i4", (3,))])
    rec["n"], rec["v"] = 3, faces
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(vbytes)
        f.write(rec.tobytes())


# reverse_imagenet_normalize (reference utils/generic_utils.py:153-159): torchvision's normalize with these
IMAGENET_REVERSE_MEAN = (-2.11790393, -2.03571429, -1.80444444)
IMAGENET_REVERSE_STD = (4.36681223, 4.46428571, 4.44444444)


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate of the fuser (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 TSDF fusion runs on CUDA (sm_90a) only; there is no CPU fallback")


class TSDFFuser:
    """Fuses depth maps into a TSDF volume (reference tools/tsdf.py:173-320)."""

    def __init__(self, tsdf: TSDF, min_depth: float = 0.5, max_depth: float = 5.0, use_gpu: bool = True):
        if not use_gpu:
            raise RuntimeError("use_gpu=False: this fuser has no CPU path")
        self.tsdf = tsdf
        self.min_depth = min_depth
        self.max_depth = max_depth
        self.use_gpu = use_gpu
        self.truncation_size = 3.0
        self.maxW = 100.0

    voxel_coords = property(lambda self: self.tsdf.voxel_coords)
    tsdf_values = property(lambda self: self.tsdf.tsdf_values)
    tsdf_weights = property(lambda self: self.tsdf.tsdf_weights)
    tsdf_colors = property(lambda self: self.tsdf.tsdf_colors)
    voxel_size = property(lambda self: self.tsdf.voxel_size)
    shape = property(lambda self: self.tsdf.tsdf_values.shape)
    truncation = property(lambda self: self.truncation_size * self.voxel_size)

    @torch.no_grad()
    def integrate_depth(self, depth_b1hw: torch.Tensor, cam_T_world_T_b44: torch.Tensor, K_b44: torch.Tensor,
                        depth_mask_b1hw: torch.Tensor | None = None, color_b3hw: torch.Tensor | None = None,
                        color_normalized: bool = True) -> None:
        """In-place update of the volume with a batch of depth maps, applied in order (:221-320).
        Inputs are taken to fp16 as ``OurFuser.fuse_frames`` does (fusers_helper.py:64-71).

        ``color_b3hw`` (required on a colour volume, refused on a plain one): (B,3,Hc,Wc) images of any
        size, taken to fp32; ``color_normalized=True`` means ImageNet-normalised as the dataloader hands
        them out (undone with ``reverse_imagenet_normalize``'s constants), False means already in [0, 1].
        The kernel picks each update's colour pixel with PyTorch's ``nearest`` rule (DESIGN §4.11)."""
        values, weights = self.tsdf.tsdf_values, self.tsdf.tsdf_weights
        colors = self.tsdf.tsdf_colors
        if colors is None and color_b3hw is not None:
            raise ValueError("color_b3hw given for a volume without colour (TSDF.from_bounds(..., color=True))")
        if colors is not None and color_b3hw is None:
            raise ValueError("this volume fuses colour: integrate_depth needs color_b3hw")
        _require_cuda(values)
        dev = values.device
        lib = _native.load()
        B, _, H, W = depth_b1hw.shape
        depth = depth_b1hw.to(dev).half().contiguous()
        E = cam_T_world_T_b44.to(dev).half().contiguous()
        K = K_b44.to(dev).half().contiguous()
        mask = None
        if depth_mask_b1hw is not None:
            mask = depth_mask_b1hw.to(dev).to(torch.uint8).contiguous()
        vol = _native.TsdfVolume()
        vol.tsdf_values, vol.tsdf_weights = values.data_ptr(), weights.data_ptr()
        vol.X, vol.Y, vol.Z = (int(d) for d in values.shape)
        for i in range(3):
            vol.origin[i] = float(self.tsdf.origin[i])
        vol.voxel_size, vol.truncation_voxels, vol.max_weight = self.voxel_size, self.truncation_size, self.maxW
        fr = _native.TsdfFrames(depth.data_ptr(), E.data_ptr(), K.data_ptr(),
                                mask.data_ptr() if mask is not None else None, B, H, W,
                                float(self.min_depth), float(self.max_depth))
        col = None
        if colors is not None:
            if color_b3hw.dim() != 4 or color_b3hw.shape[0] != B or color_b3hw.shape[1] != 3:
                raise ValueError(f"color_b3hw must be ({B}, 3, Hc, Wc), got {tuple(color_b3hw.shape)}")
            image = color_b3hw.to(dev).float().contiguous()
            mean, std = (IMAGENET_REVERSE_MEAN, IMAGENET_REVERSE_STD) if color_normalized else ((0.0,) * 3, (1.0,) * 3)
            col = _native.TsdfColor(colors.data_ptr(), image.data_ptr(), int(image.shape[2]), int(image.shape[3]),
                                    (C.c_float * 3)(*mean), (C.c_float * 3)(*std))
        with torch.cuda.device(dev):
            n = lib.srcv_tsdf_workspace_bytes(C.byref(fr))
            ws = torch.empty(n, device=dev, dtype=torch.uint8)
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            if col is not None:
                _native.check(lib.srcv_tsdf_integrate_color_f16(C.byref(vol), C.byref(fr), C.byref(col),
                                                                C.c_void_p(ws.data_ptr()), n, stream))
            else:
                _native.check(lib.srcv_tsdf_integrate_f16(C.byref(vol), C.byref(fr), C.c_void_p(ws.data_ptr()), n,
                                                          stream))
