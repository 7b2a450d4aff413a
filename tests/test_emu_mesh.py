"""CPU: the marching-cubes mesh extraction kernel (csrc/srcv_mesh.cuh) compiled for the host (tests/emu),
through TSDF.extract_mesh / to_mesh / save / from_mesh, against the fp64 oracle (oracle/mesh_oracle.py);
the C ABI's argument checks; install(fusion=True) and OurFuser's call sequence."""
import contextlib
import ctypes as C
import importlib
import sys
import types

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as M
from oracle import tsdf_oracle as T
from simplerecon_b200 import _native, tsdf as tsdf_mod
from simplerecon_b200.synthetic import make_tsdf_case
from tests import emu

install_mod = importlib.import_module("simplerecon_b200.install")   # the package exports the function


@pytest.fixture()
def emulated(monkeypatch):
    lib = emu.load_or_skip()
    monkeypatch.setattr(_native, "_lib", lib)
    monkeypatch.setattr(tsdf_mod, "_require_cuda", lambda t: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: types.SimpleNamespace(cuda_stream=0))
    real_empty = torch.empty

    def aligned_empty(*size, **kw):
        if kw.get("dtype") is torch.uint8 and len(size) == 1 and isinstance(size[0], int):
            buf = real_empty(size[0] + 256, **kw)
            off = (-buf.data_ptr()) % 256
            return buf[off:off + size[0]]
        return real_empty(*size, **kw)

    monkeypatch.setattr(torch, "empty", aligned_empty)
    return lib


def check_against_oracle(vol, scale_to_world, single_mesh):
    verts, faces, normals = vol.extract_mesh(scale_to_world=scale_to_world, single_mesh=single_mesh)
    origin_h = vol.origin.half().double().numpy()
    ov, of, on = M.extract(vol.tsdf_values, vol.tsdf_weights, scale_to_world=scale_to_world, single_mesh=single_mesh,
                           origin=origin_h, voxel_size=vol.voxel_size)
    assert verts.dtype == torch.float32 and normals.dtype == torch.float32 and faces.dtype == torch.int32
    assert verts.shape == ov.shape and normals.shape == on.shape
    assert np.array_equal(faces.numpy().astype(np.int64), of)
    kv = verts.numpy().astype(np.float64)
    mag = np.abs(ov)
    if scale_to_world:   # the fp32 terms of origin + v * voxel_size, not only their (possibly cancelling) sum
        mag = np.maximum(np.maximum(mag, np.abs(origin_h)[None]), np.abs(ov - origin_h[None]))
    tol = 4 * np.spacing(mag.astype(np.float32)).astype(np.float64)
    assert (np.abs(kv - ov) <= tol).all(), np.abs(kv - ov).max()
    assert np.abs(normals.numpy() - on).max(initial=0.0) <= 1e-5
    return verts, faces, normals


def _sphere_volume(n, c, r, origin=(0.0, 0.0, 0.0), voxel=1.0):
    x, y, z = np.meshgrid(*[np.arange(k, dtype=np.float64) for k in n], indexing="ij")
    f = (np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - r) / 3.0
    values = torch.from_numpy(np.clip(f, -1, 1)).half()
    weights = (torch.from_numpy(np.abs(f) < 2.0)).half()       # observed shell around the surface
    return tsdf_mod.TSDF(values, weights, voxel, torch.tensor(origin, dtype=torch.float32))


@pytest.mark.parametrize("dims", [(21, 19, 23), (20, 18, 24), (13, 11, 37)])   # scalar path, vector path, odd
@pytest.mark.parametrize("scale_to_world,single_mesh", [(False, False), (True, False), (False, True), (True, True)])
def test_analytic_field_matches_oracle(emulated, dims, scale_to_world, single_mesh):
    vol = _sphere_volume(dims, [d / 2 - 0.37 for d in dims], min(dims) / 2 - 3.2, origin=(-1.3, 2.7, 0.45), voxel=0.04)
    verts, faces, _ = check_against_oracle(vol, scale_to_world, single_mesh)
    assert len(faces) > 100


def _fused_room(seed, voxel, frames=2):
    c = make_tsdf_case(seed=seed, frames=frames, voxel_size=voxel, height=48, width=64)
    vol = tsdf_mod.TSDF.from_bounds(c["bounds"], voxel, device="cpu")
    tsdf_mod.TSDFFuser(vol, max_depth=c["max_depth"]).integrate_depth(c["depth"], c["cam_T_world"], c["K"])
    return vol


@pytest.mark.parametrize("scale_to_world,single_mesh", [(True, False), (False, True), (True, True)])
def test_fused_room_matches_oracle(emulated, scale_to_world, single_mesh):
    """A room fused by the emulated integration kernel: -1 where unobserved, exact zeros present."""
    vol = _fused_room(31, 0.08)
    assert int((vol.tsdf_values == 0).sum()) > 0 and int((vol.tsdf_weights == 0).sum()) > 0
    verts, faces, _ = check_against_oracle(vol, scale_to_world, single_mesh)
    assert len(faces) > 1000
    if not single_mesh:
        assert len(verts) == M.crossing_edges_torch(vol.tsdf_values)


def test_single_mesh_drops_the_unobserved_walls(emulated):
    vol = _fused_room(32, 0.09)
    _, f_all, _ = vol.extract_mesh(scale_to_world=False)
    v1, f1, _ = vol.extract_mesh(scale_to_world=False, single_mesh=True)
    assert 0 < len(f1) < len(f_all)
    # no face of a cube with a zero-weight corner: every face's vertices lie in a fully weighted cube
    assert every_face_in_a_weighted_cube(vol.tsdf_weights, v1.numpy(), f1.numpy())


def every_face_in_a_weighted_cube(weights, verts, faces) -> bool:
    """Each face lies in some cube (anchor c with c <= every vertex <= c + 1) whose 8 corners have weight."""
    w = (weights.float() > 0).cpu().numpy()
    p = verts[faces.astype(np.int64)]
    lo, hi = np.floor(p.min(1)).astype(np.int64), np.ceil(p.max(1) - 1).astype(np.int64)
    found = np.zeros(len(p), bool)
    for cx in (0, 1):
        for cy in (0, 1):
            for cz in (0, 1):
                c = lo - np.array([cx, cy, cz])
                cand = (c >= hi).all(1) & (c >= 0).all(1) & (c < np.array(w.shape) - 1).all(1)
                cc = np.where(cand[:, None], c, 0)
                ok = cand.copy()
                for d in range(8):
                    ok &= w[cc[:, 0] + (d & 1), cc[:, 1] + ((d >> 1) & 1), cc[:, 2] + (d >> 2)]
                found |= ok
    return bool(found.all())


def test_exact_zero_field(emulated):
    x, y, z = np.meshgrid(*[np.arange(k, dtype=np.float64) for k in (22, 17, 19)], indexing="ij")
    f = np.round(np.clip(np.sin(x / 3.1) + np.cos(y / 2.7) + np.sin(z / 3.7 + 0.4) - 0.2, -1, 1) * 4) / 4
    vol = tsdf_mod.TSDF(torch.from_numpy(f).half(), torch.ones(f.shape).half(), 0.05, torch.zeros(3))
    assert int((vol.tsdf_values == 0).sum()) > 200
    verts, faces, normals = check_against_oracle(vol, False, False)
    assert torch.isfinite(verts).all() and torch.isfinite(normals).all()
    assert len(verts) == M.crossing_edges_torch(vol.tsdf_values)
    p = verts[faces.long()]
    assert not ((p[:, 0] == p[:, 1]).all(-1) | (p[:, 1] == p[:, 2]).all(-1) | (p[:, 0] == p[:, 2]).all(-1)).any()


@pytest.mark.parametrize("values", [[[[-0.5, 0.5], [0.5, 0.5]], [[0.5, 0.5], [0.5, 0.5]]], None, 0.3, -1.0])
def test_tiny_and_uniform_volumes(emulated, values):
    if values is None:            # 2x2x2 with no crossing
        v = torch.full((2, 2, 2), 0.25).half()
    elif isinstance(values, float):
        v = torch.full((16, 9, 8), values).half()
    else:
        v = torch.tensor(values).half()
    vol = tsdf_mod.TSDF(v, torch.ones_like(v), 0.1, torch.zeros(3))
    for single in (False, True):
        verts, faces, normals = check_against_oracle(vol, True, single)
        if not isinstance(values, list):
            assert verts.shape == (0, 3) and faces.shape == (0, 3) and normals.shape == (0, 3)
        else:
            assert verts.shape == (3, 3) and faces.shape == (1, 3)


def _args(v, w=None, single=0, X=None):
    a = _native.MeshArgs()
    a.tsdf_values = v.data_ptr() if v is not None else None
    a.tsdf_weights = w.data_ptr() if w is not None else None
    a.X, a.Y, a.Z = (X if X is not None else v.shape[0]), v.shape[1], v.shape[2]
    a.voxel_size, a.scale_to_world, a.single_mesh = 0.1, 1, single
    return a


def test_argument_checks(emulated):
    lib = emulated
    v = torch.linspace(-1, 1, 6 * 5 * 8).reshape(6, 5, 8).half()
    a = _args(v)
    n = lib.srcv_mesh_workspace_bytes(C.byref(a))
    assert n >= 4 * v.numel()
    buf = torch.empty(n + 256, dtype=torch.uint8)
    ws = buf[(-buf.data_ptr()) % 256:][:n]
    counts = torch.zeros(2, dtype=torch.int64)
    p = lambda t: C.c_void_p(t.data_ptr())
    assert lib.srcv_mesh_count(None, p(counts), p(ws), n, None) == 1
    assert lib.srcv_mesh_count(C.byref(_args(v, X=1)), p(counts), p(ws), n, None) == 2
    assert lib.srcv_mesh_workspace_bytes(C.byref(_args(v, X=1))) == 0
    assert lib.srcv_mesh_count(C.byref(_args(v, single=1)), p(counts), p(ws), n, None) == 1   # no weights
    assert lib.srcv_mesh_count(C.byref(a), None, p(ws), n, None) == 1
    assert lib.srcv_mesh_count(C.byref(a), p(counts), p(ws), n - 256, None) == 3
    assert lib.srcv_mesh_count(C.byref(a), p(counts), p(ws), n, None) == 0
    V, F = counts.tolist()
    assert V > 0 and F > 0
    verts, normals = torch.empty(V, 3), torch.empty(V, 3)
    faces = torch.empty(F, 3, dtype=torch.int32)
    ext = lambda V_, F_, vp=p(verts), fp=p(faces): lib.srcv_mesh_extract(C.byref(a), vp, p(normals), fp, V_, F_, p(ws), n, None)
    assert ext(V + 1, F) == 2 and b"do not match" in lib.srcv_last_error()
    assert ext(V, F - 1) == 2
    assert ext(V, F, vp=None) == 1
    assert ext(V, F, fp=None) == 1
    assert ext(2 ** 31, F) == 4 and b"overflow" in lib.srcv_last_error()
    assert ext(-1, F) == 2
    n0 = lib.srcv_launch_count()
    assert ext(V, F) == 0
    assert lib.srcv_launch_count() - n0 == 2 and lib.srcv_last_variant() == b"tsdf_mesh_mc"
    with pytest.raises(_native.SrcvError):
        _native.check(ext(V + 1, F))


def read_ply(path):
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode().splitlines()
    assert header[:2] == ["ply", "format binary_little_endian 1.0"]
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in header if h.startswith("element face")).split()[-1])
    assert "property list uchar int vertex_indices" in header
    verts = np.frombuffer(data, "<f4", nv * 3, end).reshape(nv, 3)
    rec = np.frombuffer(data, [("n", "u1"), ("v", "<i4", (3,))], nf, end + 12 * nv)
    assert (rec["n"] == 3).all() and end + 12 * nv + 13 * nf == len(data)
    return verts, rec["v"]


def test_save_writes_the_extracted_mesh(emulated, tmp_path):
    vol = _sphere_volume((18, 17, 16), (8.6, 8.2, 7.9), 5.3, origin=(0.5, -1.0, 2.0), voxel=0.05)
    vol.save(str(tmp_path / "out"), "scene0000.bin")
    pv, pf = read_ply(tmp_path / "out" / "scene0000.ply")
    verts, faces, _ = vol.extract_mesh()
    assert np.array_equal(pv, verts.numpy()) and np.array_equal(pf, faces.numpy())
    assert vol.tsdf_values.device.type == "cpu"   # (the emulation's volume lives on the host anyway)


def test_to_mesh_without_trimesh_points_to_the_alternatives(emulated, monkeypatch):
    monkeypatch.setitem(sys.modules, "trimesh", None)
    vol = _sphere_volume((10, 10, 10), (4.5, 4.5, 4.5), 2.7)
    with pytest.raises(ImportError, match="extract_mesh"):
        vol.to_mesh()


class _Recorder:
    """Stands in for trimesh.Trimesh: records the constructor call."""
    calls = []

    def __init__(self, vertices=None, faces=None, normals=None):
        self.vertices, self.faces, self.normals = vertices, faces, normals
        _Recorder.calls.append(self)


def _fake_reference(monkeypatch):
    """tools / tools.tsdf / tools.fusers_helper and modules.cost_volume stand-ins."""
    ref_tsdf = types.ModuleType("tools.tsdf")
    ref_tsdf.TSDF, ref_tsdf.TSDFFuser = type("TSDF", (), {}), type("TSDFFuser", (), {})
    fh = types.ModuleType("tools.fusers_helper")
    fh.TSDF, fh.TSDFFuser = ref_tsdf.TSDF, ref_tsdf.TSDFFuser
    tools = types.ModuleType("tools")
    tools.tsdf, tools.fusers_helper = ref_tsdf, fh
    cv = types.ModuleType("modules.cost_volume")
    modules = types.ModuleType("modules")
    modules.cost_volume = cv
    for name, mod in {"tools": tools, "tools.tsdf": ref_tsdf, "tools.fusers_helper": fh, "modules": modules,
                      "modules.cost_volume": cv}.items():
        monkeypatch.setitem(sys.modules, name, mod)
    return ref_tsdf, fh


def test_install_fusion_patches_and_restores(monkeypatch):
    ref_tsdf, fh = _fake_reference(monkeypatch)
    orig = (ref_tsdf.TSDF, ref_tsdf.TSDFFuser)
    try:
        patched = install_mod.install(fusion=True)
        assert "tools.tsdf" in patched and "tools.fusers_helper" in patched
        for mod in (ref_tsdf, fh):
            assert mod.TSDF is tsdf_mod.TSDF and mod.TSDFFuser is tsdf_mod.TSDFFuser
    finally:
        install_mod.uninstall()
    for mod in (ref_tsdf, fh):
        assert (mod.TSDF, mod.TSDFFuser) == orig


def test_our_fuser_call_sequence(emulated, monkeypatch):
    """What OurFuser does (tools/fusers_helper.py:48-82): TSDF.from_mesh(gt_mesh, voxel_size),
    TSDFFuser(tsdf, max_depth), integrate_depth on .half() inputs, to_mesh(export_single_mesh=True)."""
    monkeypatch.setitem(sys.modules, "trimesh", types.SimpleNamespace(Trimesh=_Recorder))
    c = make_tsdf_case(seed=33, frames=2, voxel_size=0.1, height=48, width=64)
    corners = np.array([[c["bounds"][f"{a}min"] + 0.3, c["bounds"][f"{a}max"] - 0.3] for a in "xyz"])
    gt_mesh = types.SimpleNamespace(vertices=np.stack(np.meshgrid(*corners, indexing="ij"), -1).reshape(-1, 3))
    tsdf = tsdf_mod.TSDF.from_mesh(gt_mesh, voxel_size=0.1, device="cpu")
    fuser = tsdf_mod.TSDFFuser(tsdf, max_depth=3.0)
    fuser.integrate_depth(depth_b1hw=c["depth"].half(), cam_T_world_T_b44=c["cam_T_world"].half(), K_b44=c["K"].half())
    _Recorder.calls.clear()
    mesh = fuser.tsdf.to_mesh(export_single_mesh=True)
    assert _Recorder.calls == [mesh]
    verts, faces, normals = tsdf.extract_mesh(single_mesh=True)
    assert len(mesh.faces) > 100
    assert np.array_equal(mesh.vertices, verts.numpy()) and np.array_equal(mesh.faces, faces.numpy())
    assert np.array_equal(mesh.normals, normals.numpy())
    # from_mesh: bounds = vertex extent +- 3 voxels, then from_bounds
    pad = 3 * 0.1
    tv, _, origin = T.new_volume({"xmin": corners[0, 0] - pad, "xmax": corners[0, 1] + pad, "ymin": corners[1, 0] - pad,
                                  "ymax": corners[1, 1] + pad, "zmin": corners[2, 0] - pad, "zmax": corners[2, 1] + pad}, 0.1)
    assert tuple(tv.shape) == tuple(tsdf.tsdf_values.shape) and torch.allclose(origin, tsdf.origin)
