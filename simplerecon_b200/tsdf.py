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
        return _to_trimesh(self, self.tsdf_colors is not None, scale_to_world, export_single_mesh)

    def save(self, savepath, filename, save_mesh: bool = True):
        """Writes the mesh to ``savepath/filename`` with ``.bin`` replaced by ``.ply`` (:159-168):
        binary little-endian PLY, float x/y/z vertices, uchar-counted int faces.  Unlike the
        reference this does not move the volume to the CPU, and it needs no trimesh.  A colour volume
        adds uchar red / green / blue vertex properties."""
        _save_ply(self, self.tsdf_colors is not None, savepath, filename, save_mesh)

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


def _to_trimesh(vol, colored: bool, scale_to_world: bool, export_single_mesh: bool):
    """``to_mesh`` of a dense or voxel-block volume: its ``extract_mesh`` as a ``trimesh.Trimesh``."""
    try:
        import trimesh
    except ImportError as e:
        raise ImportError(f"{type(vol).__name__}.to_mesh needs trimesh; extract_mesh returns the mesh as tensors and "
                          "save writes a PLY file without it") from e
    if colored:                              # vertex colours as uint8 rint(255 c) (DESIGN §4.11)
        verts, faces, norms, colors = vol.extract_mesh(scale_to_world=scale_to_world, single_mesh=export_single_mesh,
                                                       with_colors=True)
        return trimesh.Trimesh(vertices=verts.cpu().numpy(), faces=faces.cpu().numpy(),
                               normals=norms.cpu().numpy(), vertex_colors=colors_to_u8(colors))
    verts, faces, norms = vol.extract_mesh(scale_to_world=scale_to_world, single_mesh=export_single_mesh)
    return trimesh.Trimesh(vertices=verts.cpu().numpy(), faces=faces.cpu().numpy(), normals=norms.cpu().numpy())


def _save_ply(vol, colored: bool, savepath, filename, save_mesh: bool) -> None:
    """``save`` of a dense or voxel-block volume: its world-space mesh as a binary PLY."""
    os.makedirs(savepath, exist_ok=True)
    if save_mesh:
        path = os.path.join(savepath, filename).replace(".bin", ".ply")
        if colored:
            verts, faces, _, colors = vol.extract_mesh(with_colors=True)
            write_ply(path, verts.cpu().numpy(), faces.cpu().numpy(), colors_to_u8(colors))
        else:
            verts, faces, _ = vol.extract_mesh()
            write_ply(path, verts.cpu().numpy(), faces.cpu().numpy())


# the reference fuser's bounds when no ground-truth mesh gives tighter ones (tools/fusers_helper.py:51-60)
DEFAULT_BOUNDS = {"xmin": -10.0, "xmax": 10.0, "ymin": -10.0, "ymax": 10.0, "zmin": -10.0, "zmax": 10.0}


class SparseCapacityError(RuntimeError):
    """A ``SparseTSDF`` ran out of block or hash capacity; ``needed`` is the ``max_blocks`` to ask for."""

    def __init__(self, message: str, needed: int):
        super().__init__(message)
        self.needed = needed


class SparseTSDF:
    """A TSDF volume without bounds (DESIGN §4.16): the dense ``TSDF``'s lattice and arithmetic, stored as
    8^3-voxel blocks in a GPU hash table, allocated only where some frame can change a voxel.

    Fed the same frames, it reads back bitwise equal to a dense ``TSDF`` on the same lattice (same
    ``origin`` and ``voxel_size``) that covers every frustum: values, weights and colours at every voxel,
    and the same mesh.  Memory is ``max_blocks`` blocks allocated up front: 2 KiB per block (values and
    weights), 8 KiB with ``color=True``, plus 24 bytes of hash table per block.  ``origin`` fixes the
    lattice; the default is the reference's ±10 m cube's corner, so the lattice is the one the reference
    fuses into without a ground-truth mesh.

    Running out of capacity neither corrupts memory nor synchronises: ``to_mesh``, ``extract_mesh``,
    ``save`` and ``to_dense`` raise a ``SparseCapacityError`` naming the ``max_blocks`` needed."""

    BLOCK = 8

    def __init__(self, voxel_size: float, origin=None, max_blocks: int = 1 << 17, color: bool = False,
                 device="cuda"):
        self.voxel_size = float(voxel_size)
        if origin is None:
            origin = [DEFAULT_BOUNDS["xmin"], DEFAULT_BOUNDS["ymin"], DEFAULT_BOUNDS["zmin"]]
        self.origin = torch.as_tensor(origin, dtype=torch.float32).detach().cpu().reshape(3).clone()
        self.max_blocks = int(max_blocks)
        self.color = bool(color)
        lib = _native.load()
        n = lib.srcv_sparse_tsdf_state_bytes(C.byref(self._desc(None)))
        if n == 0:
            raise ValueError(f"max_blocks = {self.max_blocks} is outside 1 .. 2^26")
        self.state = torch.empty(n, dtype=torch.uint8, device=device)
        _require_cuda(self.state)
        with torch.cuda.device(self.state.device):
            _native.check(lib.srcv_sparse_tsdf_reset(C.byref(self._desc()), self._stream()))

    @classmethod
    def from_bounds(cls, bounds: dict, voxel_size: float, device="cuda", color: bool = False, **kw):
        """A volume on the lattice ``TSDF.from_bounds(bounds, ...)`` would have (origin = the minimum corner)."""
        return cls(voxel_size, origin=[bounds["xmin"], bounds["ymin"], bounds["zmin"]], color=color, device=device, **kw)

    def _desc(self, state=False, truncation_voxels: float = 3.0, max_weight: float = 100.0) -> _native.SparseTsdf:
        d = _native.SparseTsdf()
        d.state = None if state is None else self.state.data_ptr()
        d.max_blocks, d.color = self.max_blocks, int(self.color)
        for i in range(3):
            d.origin[i] = float(self.origin[i])
        d.voxel_size, d.truncation_voxels, d.max_weight = self.voxel_size, truncation_voxels, max_weight
        return d

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.state.device).cuda_stream)

    def header(self) -> list[int]:
        """The state header (``SRCV_SPARSE_HDR_*``): blocks requested, lost inserts, range flags.  Syncs."""
        return [int(x) for x in self.state[:4 * _native.SPARSE_HDR_WORDS].view(torch.int32).tolist()]

    @property
    def allocated_blocks(self) -> int:
        """Blocks allocated so far (a host synchronisation)."""
        return min(self.header()[_native.SPARSE_HDR_BLOCKS], self.max_blocks)

    def _check_capacity(self, blocks: int | None = None, what: str = "") -> int:
        hdr = self.header()
        req, lost, rng = hdr[_native.SPARSE_HDR_BLOCKS], hdr[_native.SPARSE_HDR_LOST], hdr[_native.SPARSE_HDR_RANGE]
        if rng:
            raise RuntimeError("SparseTSDF: a frame reached outside voxel indices -2^23 + 8 .. 2^23 - 1 around the "
                               "origin or had a singular projection; its voxels were not fused")
        if req > self.max_blocks or lost:
            needed = max(req, self.max_blocks + 1) if not lost else max(req, self.max_blocks) * 2
            raise SparseCapacityError(
                f"SparseTSDF ran out of capacity{what}: it needs max_blocks >= {needed} "
                f"(it has {self.max_blocks}); the volume is incomplete, rebuild it with a larger max_blocks", needed)
        return req

    @torch.no_grad()
    def extract_mesh(self, scale_to_world: bool = True, single_mesh: bool = False, with_colors: bool = False):
        """``TSDF.extract_mesh`` on the unbounded lattice: the same ``(verts, faces, normals[, colors])``
        as a dense volume on this lattice covering every frustum, up to the order of vertices and faces
        (DESIGN §4.16).  Host synchronisations: the capacity checks and the vertex / face counts."""
        if with_colors and not self.color:
            raise ValueError("with_colors=True needs a colour volume (SparseTSDF(..., color=True))")
        lib = _native.load()
        dev = self.state.device
        n = self._check_capacity()
        desc = self._desc()
        with torch.cuda.device(dev):
            stream = self._stream()
            _native.check(lib.srcv_sparse_tsdf_mesh_begin(C.byref(desc), n, stream))
            try:
                nmesh = self._check_capacity(what=" for the mesh's boundary blocks")
                a = _native.SparseMeshArgs()
                a.blocks = nmesh
                origin_h = self.origin.half().float()
                for i in range(3):
                    a.origin[i] = float(origin_h[i])
                a.scale_to_world, a.single_mesh = int(bool(scale_to_world)), int(bool(single_mesh))
                nbytes = lib.srcv_sparse_tsdf_mesh_workspace_bytes(C.byref(a))
                ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
                counts = torch.empty(2, device=dev, dtype=torch.int64)
                _native.check(lib.srcv_sparse_tsdf_mesh_count(C.byref(desc), C.byref(a), C.c_void_p(counts.data_ptr()),
                                                              C.c_void_p(ws.data_ptr()), nbytes, stream))
                V, F = (int(c) for c in counts.tolist())
                verts = torch.empty((V, 3), device=dev, dtype=torch.float32)
                normals = torch.empty((V, 3), device=dev, dtype=torch.float32)
                faces = torch.empty((F, 3), device=dev, dtype=torch.int32)
                colors = torch.empty((V, 3), device=dev, dtype=torch.float32) if with_colors else None
                ptr = lambda t: C.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)
                _native.check(lib.srcv_sparse_tsdf_mesh_extract(
                    C.byref(desc), C.byref(a), ptr(verts), ptr(normals), ptr(colors) if with_colors else None,
                    ptr(faces), V, F, C.c_void_p(ws.data_ptr()), nbytes, stream))
            finally:
                _native.check(lib.srcv_sparse_tsdf_mesh_end(C.byref(desc), n, stream))
        return (verts, faces, normals, colors) if with_colors else (verts, faces, normals)

    def to_mesh(self, scale_to_world: bool = True, export_single_mesh: bool = False):
        """``TSDF.to_mesh``: a ``trimesh.Trimesh`` (vertex colours on a colour volume)."""
        self._check_capacity()
        return _to_trimesh(self, self.color, scale_to_world, export_single_mesh)

    def save(self, savepath, filename, save_mesh: bool = True):
        """``TSDF.save``: the world-space mesh as a binary PLY at ``savepath/filename`` (``.bin`` -> ``.ply``)."""
        self._check_capacity()
        _save_ply(self, self.color, savepath, filename, save_mesh)

    @torch.no_grad()
    def to_dense(self, bounds: dict) -> TSDF:
        """The dense ``TSDF`` over ``bounds``, as ``TSDF.from_bounds(bounds, voxel_size)`` lays it out but on this
        volume's lattice: the box starts at the lattice voxel at or below (xmin, ymin, zmin), and its origin is
        that voxel's position, origin + i * voxel_size in fp32 (so with ``bounds``' minimum corner on the
        origin, it is exactly ``from_bounds``' volume).  Voxels outside every allocated block read -1 / 0 / 0."""
        lib = _native.load()
        self._check_capacity()
        dims = tuple(int(np.ceil((bounds[a + "max"] - bounds[a + "min"]) / self.voxel_size / TSDF.VOX_MOD)) * TSDF.VOX_MOD
                     for a in "xyz")
        lo = [int(np.floor(np.float64(np.float32(bounds[a + "min"]) - np.float32(self.origin[i]))
                           / np.float64(np.float32(self.voxel_size)) + 1e-9)) for i, a in enumerate("xyz")]
        origin = torch.tensor([np.float32(self.origin[i]) + np.float32(lo[i]) * np.float32(self.voxel_size)
                               for i in range(3)], dtype=torch.float32)
        dev = self.state.device
        values = torch.empty(dims, dtype=torch.float16, device=dev)
        weights = torch.empty(dims, dtype=torch.float16, device=dev)
        colors = torch.empty((3, *dims), dtype=torch.float32, device=dev) if self.color else None
        with torch.cuda.device(dev):
            _native.check(lib.srcv_sparse_tsdf_read_box(
                C.byref(self._desc()), (C.c_int32 * 3)(*lo), (C.c_int32 * 3)(*dims), C.c_void_p(values.data_ptr()),
                C.c_void_p(weights.data_ptr()), C.c_void_p(colors.data_ptr()) if colors is not None else None,
                self._stream()))
        return TSDF(values, weights, self.voxel_size, origin, colors)

    def _integrate(self, fr, col, truncation_voxels: float, max_weight: float) -> None:
        lib = _native.load()
        desc = self._desc(truncation_voxels=truncation_voxels, max_weight=max_weight)
        dev = self.state.device
        with torch.cuda.device(dev):
            n = lib.srcv_sparse_tsdf_workspace_bytes(C.byref(fr))
            ws = torch.empty(n, device=dev, dtype=torch.uint8)
            stream = self._stream()
            if col is not None:
                _native.check(lib.srcv_sparse_tsdf_integrate_color_f16(C.byref(desc), C.byref(fr), C.byref(col),
                                                                       C.c_void_p(ws.data_ptr()), n, stream))
            else:
                _native.check(lib.srcv_sparse_tsdf_integrate_f16(C.byref(desc), C.byref(fr), C.c_void_p(ws.data_ptr()),
                                                                 n, stream))

    def cuda(self):
        self.state = self.state.cuda()
        return self

    def cpu(self):
        self.state = self.state.cpu()
        return self


def colors_to_u8(colors) -> np.ndarray:
    """(V,3) colours in [0, 1] -> uint8 rint(255 c) (round half to even), as a host array."""
    c = colors.detach().cpu().numpy() if torch.is_tensor(colors) else np.asarray(colors)
    return np.rint(np.float32(255.0) * np.clip(c.astype(np.float32), 0.0, 1.0)).astype(np.uint8)


def write_ply(path, verts: np.ndarray, faces: np.ndarray | None, colors: np.ndarray | None = None) -> None:
    """Binary little-endian PLY: float x, y, z (and uchar red, green, blue when ``colors`` is given:
    uint8 as is, floats in [0, 1] through ``colors_to_u8``) per vertex; a uchar count and int indices per
    face.  ``faces=None`` writes a point cloud: no face element at all (``read_ply`` returns faces=None)."""
    verts = np.ascontiguousarray(verts, dtype="<f4").reshape(-1, 3)
    if faces is not None:
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
    header = f"ply\nformat binary_little_endian 1.0\nelement vertex {len(verts)}\n{vprops}"
    fbytes = b""
    if faces is not None:
        header += f"element face {len(faces)}\nproperty list uchar int vertex_indices\n"
        rec = np.empty(len(faces), dtype=[("n", "u1"), ("v", "<i4", (3,))])
        rec["n"], rec["v"] = 3, faces
        fbytes = rec.tobytes()
    with open(path, "wb") as f:
        f.write((header + "end_header\n").encode("ascii"))
        f.write(vbytes)
        f.write(fbytes)


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2",
              "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4",
              "float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8"}


def read_ply(path):
    """``(verts (V,3) float32, faces (F,3) int64 or None)`` from a binary little-endian PLY, such as
    ``write_ply`` writes or ScanNet's ``_vh_clean_2.ply`` (float x, y, z plus uchar RGBA).

    Vertex x / y / z may be float or double; any other scalar vertex property is skipped by its size.  The
    optional face element is a list of triangles with a uchar count and int or uint indices.  Other formats
    (ASCII, big-endian) raise ``ValueError``."""
    with open(path, "rb") as fh:
        if fh.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        elements, fmt = [], None
        while True:
            line = fh.readline()
            if not line:
                raise ValueError(f"{path}: the PLY header has no end_header")
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "end_header":
                break
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == "property":
                if not elements:
                    raise ValueError(f"{path}: a property before any element")
                elements[-1][2].append(tok[1:])
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: read_ply reads binary little-endian PLY only, this file is {fmt}")
        data = fh.read()
    verts, faces, off = None, None, 0
    for name, count, props in elements:
        if any(p[0] == "list" for p in props):
            if name != "face" or len(props) != 1 or props[0][1] not in ("uchar", "uint8") or \
                    props[0][2] not in ("int", "int32", "uint", "uint32"):
                raise ValueError(f"{path}: only a face element of one list (uchar count, int or uint indices) is read")
            rec = np.dtype([("n", "u1"), ("v", _PLY_TYPES[props[0][2]], (3,))])
            arr = np.frombuffer(data, dtype=rec, count=count, offset=off)
            if count and not np.all(arr["n"] == 3):
                raise ValueError(f"{path}: only triangle faces are read")
            faces = arr["v"].astype(np.int64)
            off += rec.itemsize * count
            continue
        try:
            rec = np.dtype([(p[1], _PLY_TYPES[p[0]]) for p in props])
        except KeyError as e:
            raise ValueError(f"{path}: unknown PLY property type {e.args[0]}") from None
        if name == "vertex":
            if not all(a in rec.names for a in "xyz"):
                raise ValueError(f"{path}: the vertex element has no x, y, z")
            arr = np.frombuffer(data, dtype=rec, count=count, offset=off)
            verts = np.stack([arr[a].astype(np.float32) for a in "xyz"], 1)
        off += rec.itemsize * count
    if verts is None:
        raise ValueError(f"{path}: no vertex element")
    return verts, faces


# reverse_imagenet_normalize (reference utils/generic_utils.py:153-159): torchvision's normalize with these
IMAGENET_REVERSE_MEAN = (-2.11790393, -2.03571429, -1.80444444)
IMAGENET_REVERSE_STD = (4.36681223, 4.46428571, 4.44444444)


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate of the fuser (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 TSDF fusion runs on CUDA (sm_90a) only; there is no CPU fallback")


class TSDFFuser:
    """Fuses depth maps into a TSDF volume (reference tools/tsdf.py:173-320)."""

    def __init__(self, tsdf: TSDF | SparseTSDF, min_depth: float = 0.5, max_depth: float = 5.0, use_gpu: bool = True):
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
        The kernel picks each update's colour pixel with PyTorch's ``nearest`` rule (DESIGN §4.11).

        On a ``SparseTSDF`` the blocks the frames can reach are allocated first, on the device; nothing
        synchronises with the host (DESIGN §4.16)."""
        sparse = isinstance(self.tsdf, SparseTSDF)
        if sparse:
            colored, ref = self.tsdf.color, self.tsdf.state
        else:
            colored, ref = self.tsdf.tsdf_colors is not None, self.tsdf.tsdf_values
        if not colored and color_b3hw is not None:
            raise ValueError("color_b3hw given for a volume without colour (TSDF.from_bounds(..., color=True))")
        if colored and color_b3hw is None:
            raise ValueError("this volume fuses colour: integrate_depth needs color_b3hw")
        _require_cuda(ref)
        dev = ref.device
        lib = _native.load()
        B, _, H, W = depth_b1hw.shape
        depth = depth_b1hw.to(dev).half().contiguous()
        E = cam_T_world_T_b44.to(dev).half().contiguous()
        K = K_b44.to(dev).half().contiguous()
        mask = None
        if depth_mask_b1hw is not None:
            mask = depth_mask_b1hw.to(dev).to(torch.uint8).contiguous()
        fr = _native.TsdfFrames(depth.data_ptr(), E.data_ptr(), K.data_ptr(),
                                mask.data_ptr() if mask is not None else None, B, H, W,
                                float(self.min_depth), float(self.max_depth))
        col = None
        if colored:
            if color_b3hw.dim() != 4 or color_b3hw.shape[0] != B or color_b3hw.shape[1] != 3:
                raise ValueError(f"color_b3hw must be ({B}, 3, Hc, Wc), got {tuple(color_b3hw.shape)}")
            image = color_b3hw.to(dev).float().contiguous()
            mean, std = (IMAGENET_REVERSE_MEAN, IMAGENET_REVERSE_STD) if color_normalized else ((0.0,) * 3, (1.0,) * 3)
            planes = None if sparse else self.tsdf.tsdf_colors.data_ptr()     # a SparseTSDF keeps them in its state
            col = _native.TsdfColor(planes, image.data_ptr(), int(image.shape[2]), int(image.shape[3]),
                                    (C.c_float * 3)(*mean), (C.c_float * 3)(*std))
        if sparse:
            self.tsdf._integrate(fr, col, self.truncation_size, self.maxW)
            return
        values, weights = self.tsdf.tsdf_values, self.tsdf.tsdf_weights
        vol = _native.TsdfVolume()
        vol.tsdf_values, vol.tsdf_weights = values.data_ptr(), weights.data_ptr()
        vol.X, vol.Y, vol.Z = (int(d) for d in values.shape)
        for i in range(3):
            vol.origin[i] = float(self.tsdf.origin[i])
        vol.voxel_size, vol.truncation_voxels, vol.max_weight = self.voxel_size, self.truncation_size, self.maxW
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
