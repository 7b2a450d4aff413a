"""CPU: colour fusion (DESIGN §4.11) — the colour instantiations of the integration kernel and the vertex-colour
pass compiled for the host (tests/emu), through TSDF / TSDFFuser / ColorFuser, bit for bit against the float32
oracle (oracle/color_oracle.py); the C ABI's argument checks; coloured PLY; install(fuse_color=True)."""
import contextlib
import ctypes as C
import importlib
import sys
import types

import numpy as np
import pytest
import torch

from oracle import color_oracle as CO
from oracle import tsdf_oracle as T
from simplerecon_b200 import _native, fusers, tsdf as tsdf_mod
from simplerecon_b200.synthetic import make_color_tsdf_case, room_wall_color
from tests import emu

install_mod = importlib.import_module("simplerecon_b200.install")


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


def fuse_both(c, voxel, calls=1, zcut=None, normalized=True, batch_split=None):
    """The same frames through a colour volume (kernel), a plain volume (kernel) and the oracle."""
    vol = tsdf_mod.TSDF.from_bounds(c["bounds"], voxel, device="cpu", color=True)
    plain = tsdf_mod.TSDF.from_bounds(c["bounds"], voxel, device="cpu")
    tv, tw, origin = T.new_volume(c["bounds"], voxel)
    tc = torch.zeros((3, *tv.shape))
    if zcut is not None:   # Z % 8 != 0: the scalar path
        cut = lambda t: t[..., :zcut].contiguous()
        vol = tsdf_mod.TSDF(cut(vol.tsdf_values), cut(vol.tsdf_weights), voxel, origin, cut(vol.tsdf_colors))
        plain = tsdf_mod.TSDF(cut(plain.tsdf_values), cut(plain.tsdf_weights), voxel, origin)
        tv, tw, tc = cut(tv), cut(tw), cut(tc)
    image = c["color"] if normalized else c["color_raw"]
    mean, std = (CO.REVERSE_MEAN, CO.REVERSE_STD) if normalized else ((0.0,) * 3, (1.0,) * 3)
    fuser, pfuser = tsdf_mod.TSDFFuser(vol, max_depth=c["max_depth"]), tsdf_mod.TSDFFuser(plain, max_depth=c["max_depth"])
    for _ in range(calls):
        fuser.integrate_depth(c["depth"], c["cam_T_world"], c["K"], c["mask"], color_b3hw=image,
                              color_normalized=normalized)
        pfuser.integrate_depth(c["depth"], c["cam_T_world"], c["K"], c["mask"])
        CO.integrate(tv, tw, tc, origin, voxel, c["depth"], c["cam_T_world"], c["K"], image, c["mask"],
                     min_depth=fuser.min_depth, max_depth=c["max_depth"], mean=mean, std=std)
    return vol, plain, (tv, tw, tc)


def assert_bitwise(vol, plain, ref):
    tv, tw, tc = ref
    assert int((tw > 0).sum()) > 300
    assert torch.equal(vol.tsdf_weights, plain.tsdf_weights) and torch.equal(vol.tsdf_values, plain.tsdf_values)
    assert torch.equal(vol.tsdf_weights, tw) and torch.equal(vol.tsdf_values, tv)
    assert torch.equal(vol.tsdf_colors.view(torch.int32), tc.view(torch.int32)), (vol.tsdf_colors - tc).abs().max()
    # weight > 0 <=> the colour has been observed (no wall of the synthetic room is black)
    assert torch.equal(vol.tsdf_weights > 0, vol.tsdf_colors.sum(0) > 0)


@pytest.mark.parametrize("frames,color_hw,masked,calls", [
    (2, (72, 96), False, 2),      # 1.5x up-scaled colour (non-integer ratio)
    (2, (96, 128), True, 1),      # 2x, masked depth
    (3, (24, 32), False, 1),      # 0.5x down-scaled
    (2, (37, 53), False, 1),      # odd ratio
    (18, (48, 64), False, 1),     # more than 16 frames: two launches
])
def test_integrate_color_matches_oracle_bitwise(emulated, frames, color_hw, masked, calls):
    c = make_color_tsdf_case(seed=frames, frames=frames, voxel_size=0.1, height=48, width=64, color_hw=color_hw,
                             masked=masked)
    vol, plain, ref = fuse_both(c, 0.1, calls=calls)
    assert_bitwise(vol, plain, ref)


@pytest.mark.parametrize("normalized", [True, False])
def test_scalar_path_and_unnormalised_colour(emulated, normalized):
    c = make_color_tsdf_case(seed=9, frames=2, voxel_size=0.1, height=48, width=64, color_hw=(60, 80))
    vol, plain, ref = fuse_both(c, 0.1, zcut=29, normalized=normalized)
    assert vol.tsdf_values.shape[2] == 29
    assert_bitwise(vol, plain, ref)


def _fused_color_room(seed=11, voxel=0.08, frames=3):
    c = make_color_tsdf_case(seed=seed, frames=frames, voxel_size=voxel, height=48, width=64, color_hw=(72, 96))
    vol = tsdf_mod.TSDF.from_bounds(c["bounds"], voxel, device="cpu", color=True)
    tsdf_mod.TSDFFuser(vol, max_depth=c["max_depth"]).integrate_depth(c["depth"], c["cam_T_world"], c["K"],
                                                                       color_b3hw=c["color"])
    return vol, c


@pytest.mark.parametrize("single_mesh", [False, True])
@pytest.mark.parametrize("scale_to_world", [False, True])
def test_vertex_colors_match_oracle_bitwise(emulated, single_mesh, scale_to_world):
    vol, _ = _fused_color_room()
    v, f, n, col = vol.extract_mesh(scale_to_world=scale_to_world, single_mesh=single_mesh, with_colors=True)
    pv, pf, pn = vol.extract_mesh(scale_to_world=scale_to_world, single_mesh=single_mesh)
    assert torch.equal(v, pv) and torch.equal(f, pf) and torch.equal(n, pn)
    ref = CO.vertex_colors(vol.tsdf_values, vol.tsdf_weights, vol.tsdf_colors, single_mesh=single_mesh)
    assert col.shape == (len(v), 3) and col.dtype == torch.float32 and len(f) > 500
    assert np.array_equal(col.numpy().view(np.int32), ref.view(np.int32))
    if single_mesh:                     # every vertex of a fully weighted cube has weighted endpoints
        assert not bool((col == np.float32(0.7)).all(1).any())


def test_vertex_colors_scalar_path(emulated):
    vol, _ = _fused_color_room(seed=12, voxel=0.09)
    cut = lambda t: t[..., :21].contiguous()
    vol = tsdf_mod.TSDF(cut(vol.tsdf_values), cut(vol.tsdf_weights), vol.voxel_size, vol.origin, cut(vol.tsdf_colors))
    _, f, _, col = vol.extract_mesh(with_colors=True)
    ref = CO.vertex_colors(vol.tsdf_values, vol.tsdf_weights, vol.tsdf_colors)
    assert len(f) > 100 and np.array_equal(col.numpy().view(np.int32), ref.view(np.int32))


def test_wall_colours_reach_the_mesh(emulated):
    """Vertices more than 2 voxels from every wall edge and checker line carry their wall's analytic colour:
    90 % within 1e-4 per channel (fp32 rounding of the running average) and all within 0.1 (a voxel seen at
    a grazing angle samples the wall up to a few voxels away along the ray, so near a checker line some
    updates average in the neighbouring cell's colour)."""
    voxel = 0.05
    c = make_color_tsdf_case(seed=13, frames=4, voxel_size=voxel, height=60, width=80, color_hw=(90, 120))
    vol = tsdf_mod.TSDF.from_bounds(c["bounds"], voxel, device="cpu", color=True)
    tsdf_mod.TSDFFuser(vol, max_depth=c["max_depth"]).integrate_depth(c["depth"], c["cam_T_world"], c["K"],
                                                                       color_b3hw=c["color"])
    check_wall_colors(vol, voxel)


def check_wall_colors(vol, voxel):
    v, _, _, col = vol.extract_mesh(single_mesh=True, with_colors=True)
    rgb, _, edge, line = room_wall_color(v.cpu().double())
    keep = (edge > 2 * voxel) & (line > 2 * voxel)
    assert int(keep.sum()) > 200
    err = (col.cpu().double()[keep] - rgb[keep]).abs().max(1).values
    assert float((err <= 1e-4).double().mean()) >= 0.9, float((err <= 1e-4).double().mean())
    assert float(err.max()) <= 0.1, float(err.max())


def test_argument_checks(emulated):
    c = make_color_tsdf_case(seed=3, frames=1, voxel_size=0.1, height=24, width=32, color_hw=(24, 32))
    plain = tsdf_mod.TSDF.from_bounds(c["bounds"], 0.1, device="cpu")
    colored = tsdf_mod.TSDF.from_bounds(c["bounds"], 0.1, device="cpu", color=True)
    with pytest.raises(ValueError, match="without colour"):
        tsdf_mod.TSDFFuser(plain).integrate_depth(c["depth"], c["cam_T_world"], c["K"], color_b3hw=c["color"])
    with pytest.raises(ValueError, match="needs color_b3hw"):
        tsdf_mod.TSDFFuser(colored).integrate_depth(c["depth"], c["cam_T_world"], c["K"])
    with pytest.raises(ValueError, match="3, Hc, Wc"):
        tsdf_mod.TSDFFuser(colored).integrate_depth(c["depth"], c["cam_T_world"], c["K"], color_b3hw=c["color"][:, :2])
    with pytest.raises(ValueError, match="with_colors"):
        plain.extract_mesh(with_colors=True)
    with pytest.raises(ValueError, match=r"\(3, X, Y, Z\)"):
        tsdf_mod.TSDF(plain.tsdf_values, plain.tsdf_weights, 0.1, plain.origin, colors=torch.zeros(3, 2, 2, 2))
    # fp16 / bf16 images are taken to fp32 in Python
    tsdf_mod.TSDFFuser(colored, max_depth=3.0).integrate_depth(c["depth"], c["cam_T_world"], c["K"],
                                                                color_b3hw=c["color"].bfloat16())
    assert int((colored.tsdf_weights > 0).sum()) > 0


def test_c_abi_argument_checks(emulated):
    lib = emulated
    c = make_color_tsdf_case(seed=4, frames=1, voxel_size=0.1, height=24, width=32, color_hw=(30, 40))
    vol = tsdf_mod.TSDF.from_bounds(c["bounds"], 0.1, device="cpu", color=True)
    depth, E, K = c["depth"].half().contiguous(), c["cam_T_world"].half().contiguous(), c["K"].half().contiguous()
    image = c["color"].contiguous()
    v = _native.TsdfVolume()
    v.tsdf_values, v.tsdf_weights = vol.tsdf_values.data_ptr(), vol.tsdf_weights.data_ptr()
    v.X, v.Y, v.Z = vol.tsdf_values.shape
    v.voxel_size, v.truncation_voxels, v.max_weight = 0.1, 3.0, 100.0
    fr = _native.TsdfFrames(depth.data_ptr(), E.data_ptr(), K.data_ptr(), None, 1, 24, 32, 0.5, 3.0)
    n = lib.srcv_tsdf_workspace_bytes(C.byref(fr))
    buf = torch.empty(n + 256, dtype=torch.uint8)
    ws = C.c_void_p(buf[(-buf.data_ptr()) % 256:].data_ptr())
    col = lambda **kw: _native.TsdfColor(kw.get("colors", vol.tsdf_colors.data_ptr()), kw.get("images", image.data_ptr()),
                                         kw.get("Hc", 30), kw.get("Wc", 40), (C.c_float * 3)(0, 0, 0),
                                         (C.c_float * 3)(*kw.get("std", (1, 1, 1))))
    run = lambda cl, vv=v: lib.srcv_tsdf_integrate_color_f16(C.byref(vv), C.byref(fr), cl, ws, n, None)
    assert run(None) == 1
    assert run(C.byref(col(colors=None))) == 1
    assert run(C.byref(col(images=None))) == 1
    assert run(C.byref(col(Hc=0))) == 2 and b"Hc" in lib.srcv_last_error()
    assert run(C.byref(col(Wc=-3))) == 2
    assert run(C.byref(col(std=(1, 0, 1)))) == 2
    assert run(C.byref(col(colors=vol.tsdf_colors.data_ptr() + 2))) == 4
    assert lib.srcv_tsdf_integrate_color_f16(C.byref(v), None, C.byref(col()), ws, n, None) == 1
    bad = _native.TsdfVolume.from_buffer_copy(v)
    bad.X = 0
    assert run(C.byref(col()), bad) == 2
    assert run(C.byref(col())) == 0 and lib.srcv_last_variant() == b"tsdf_integrate_color_f16"
    # mesh: the colour extraction refuses what it needs and is missing
    a = _native.MeshArgs()
    a.tsdf_values, a.tsdf_weights = vol.tsdf_values.data_ptr(), vol.tsdf_weights.data_ptr()
    a.X, a.Y, a.Z = vol.tsdf_values.shape
    a.voxel_size, a.scale_to_world = 0.1, 1
    m = lib.srcv_mesh_workspace_bytes(C.byref(a))
    mb = torch.empty(m + 256, dtype=torch.uint8)
    mws = C.c_void_p(mb[(-mb.data_ptr()) % 256:].data_ptr())
    counts = torch.zeros(2, dtype=torch.int64)
    assert lib.srcv_mesh_count(C.byref(a), C.c_void_p(counts.data_ptr()), mws, m, None) == 0
    V, F = counts.tolist()
    assert V > 0
    verts, normals, vc = torch.empty(V, 3), torch.empty(V, 3), torch.empty(V, 3)
    faces = torch.empty(F, 3, dtype=torch.int32)
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    ext = lambda aa=a, colors=vol.tsdf_colors, vcol=vc, V_=V: lib.srcv_mesh_extract_color(
        C.byref(aa), p(colors), p(verts), p(normals), p(vcol), p(faces), V_, F, mws, m, None)
    assert ext(colors=None) == 1
    assert ext(vcol=None) == 1
    nw = _native.MeshArgs.from_buffer_copy(a)
    nw.tsdf_weights = None
    assert ext(aa=nw) == 1
    assert ext(V_=V + 1) == 2
    n0 = lib.srcv_launch_count()
    assert ext() == 0 and lib.srcv_last_variant() == b"tsdf_mesh_mc_color"
    assert lib.srcv_launch_count() - n0 == 3


def read_ply(path):
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode().splitlines()
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in header if h.startswith("element face")).split()[-1])
    colored = "property uchar red" in header
    vdt = [("p", "<f4", (3,))] + ([("c", "u1", (3,))] if colored else [])
    vrec = np.frombuffer(data, vdt, nv, end)
    rec = np.frombuffer(data, [("n", "u1"), ("v", "<i4", (3,))], nf, end + vrec.itemsize * nv)
    assert (rec["n"] == 3).all() and end + vrec.itemsize * nv + 13 * nf == len(data)
    return header, vrec["p"], rec["v"], (vrec["c"] if colored else None)


def test_ply_round_trip_and_plain_bytes(emulated, tmp_path):
    vol, _ = _fused_color_room(seed=14, voxel=0.1, frames=2)
    vol.save(str(tmp_path), "scene.bin")
    header, pv, pf, pc = read_ply(tmp_path / "scene.ply")
    assert header[3:9] == ["property float x", "property float y", "property float z", "property uchar red",
                           "property uchar green", "property uchar blue"]
    v, f, _, col = vol.extract_mesh(with_colors=True)
    assert np.array_equal(pv, v.numpy()) and np.array_equal(pf, f.numpy())
    assert np.array_equal(pc, np.rint(np.float32(255) * col.numpy()).astype(np.uint8))
    # a plain volume's save: the bytes the plain writer always produced
    plain = tsdf_mod.TSDF(vol.tsdf_values, vol.tsdf_weights, vol.voxel_size, vol.origin)
    plain.save(str(tmp_path), "plain.bin")
    pv2, pf2 = v.numpy(), f.numpy()
    rec = np.empty(len(pf2), dtype=[("n", "u1"), ("v", "<i4", (3,))])
    rec["n"], rec["v"] = 3, pf2
    expect = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(pv2)}\nproperty float x\nproperty float y\n"
              f"property float z\nelement face {len(pf2)}\nproperty list uchar int vertex_indices\nend_header\n"
              ).encode() + pv2.astype("<f4").tobytes() + rec.tobytes()
    assert (tmp_path / "plain.ply").read_bytes() == expect
    tsdf_mod.write_ply(tmp_path / "f.ply", pv2, pf2, col.numpy())       # floats -> rint(255 c)
    assert np.array_equal(read_ply(tmp_path / "f.ply")[3], pc)
    with pytest.raises(ValueError, match="colours for"):
        tsdf_mod.write_ply(tmp_path / "g.ply", pv2, pf2, pc[:-1])


class _Recorder:
    calls = []

    def __init__(self, vertices=None, faces=None, normals=None, vertex_colors=None):
        self.vertices, self.faces, self.normals, self.vertex_colors = vertices, faces, normals, vertex_colors
        _Recorder.calls.append(self)


def test_to_mesh_colours_and_plain_call(emulated, monkeypatch):
    monkeypatch.setitem(sys.modules, "trimesh", types.SimpleNamespace(Trimesh=_Recorder))
    vol, _ = _fused_color_room(seed=15, voxel=0.1, frames=2)
    mesh = vol.to_mesh(export_single_mesh=True)
    v, f, n, col = vol.extract_mesh(single_mesh=True, with_colors=True)
    assert mesh.vertex_colors.dtype == np.uint8 and mesh.vertex_colors.shape == (len(v), 3)
    assert np.array_equal(mesh.vertex_colors, np.rint(np.float32(255) * col.numpy()).astype(np.uint8))
    assert np.array_equal(mesh.vertices, v.numpy()) and np.array_equal(mesh.faces, f.numpy())
    calls = []
    monkeypatch.setitem(sys.modules, "trimesh", types.SimpleNamespace(Trimesh=lambda **kw: calls.append(kw)))
    tsdf_mod.TSDF(vol.tsdf_values, vol.tsdf_weights, vol.voxel_size, vol.origin).to_mesh()
    assert sorted(calls[0]) == ["faces", "normals", "vertices"]          # exactly as before on a plain volume


def _fake_reference(monkeypatch):
    """tools / tools.tsdf / tools.fusers_helper / modules.cost_volume stand-ins; get_fuser records its calls."""
    ref_tsdf = types.ModuleType("tools.tsdf")
    ref_tsdf.TSDF, ref_tsdf.TSDFFuser = type("TSDF", (), {}), type("TSDFFuser", (), {})
    fh = types.ModuleType("tools.fusers_helper")
    fh.TSDF, fh.TSDFFuser = ref_tsdf.TSDF, ref_tsdf.TSDFFuser
    fh.calls = []
    fh.get_fuser = lambda opts, scan: fh.calls.append((opts, scan)) or "original"
    fh.ScannetDataset = types.SimpleNamespace(get_gt_mesh_path=lambda root, split, scan: f"{root}/{split}/{scan}.ply")
    tools = types.ModuleType("tools")
    tools.tsdf, tools.fusers_helper = ref_tsdf, fh
    cv = types.ModuleType("modules.cost_volume")
    modules = types.ModuleType("modules")
    modules.cost_volume = cv
    for name, mod in {"tools": tools, "tools.tsdf": ref_tsdf, "tools.fusers_helper": fh, "modules": modules,
                      "modules.cost_volume": cv}.items():
        monkeypatch.setitem(sys.modules, name, mod)
    return ref_tsdf, fh


def _opts(**kw):
    base = dict(dataset="scannet", dataset_path="/data", split="test", depth_fuser="ours", fuse_color=True,
                fusion_resolution=0.04, fusion_max_depth=3.0)
    return types.SimpleNamespace(**{**base, **kw})


def test_install_fuse_color_redirects_ours_and_delegates_the_rest(monkeypatch):
    _, fh = _fake_reference(monkeypatch)
    orig = fh.get_fuser
    made = []
    monkeypatch.setattr(fusers, "ColorFuser", lambda **kw: made.append(kw) or "color")
    with pytest.raises(ValueError, match="fusion=True"):
        install_mod.install(fuse_color=True)
    try:
        install_mod.install(fusion=True, fuse_color=True)
        assert fh.get_fuser is not orig and fh.TSDF is tsdf_mod.TSDF
        assert fh.get_fuser(_opts(), "scene0707_00") == "color"
        assert made == [dict(gt_path="/data/test/scene0707_00.ply", fusion_resolution=0.04, max_fusion_depth=3.0,
                             fuse_color=True)]
        assert fh.get_fuser(_opts(dataset="7scenes"), "s") == "color" and made[-1]["gt_path"] is None
        for kw in (dict(fuse_color=False), dict(depth_fuser="open3d"), dict(depth_fuser="open3d", fuse_color=False),
                   dict(depth_fuser="nope")):
            o = _opts(**kw)
            assert fh.get_fuser(o, "scan") == "original" and fh.calls[-1] == (o, "scan")
        assert len(fh.calls) == 4 and len(made) == 2
    finally:
        install_mod.uninstall()
    assert fh.get_fuser is orig
    # install(fusion=True) alone leaves get_fuser alone
    try:
        install_mod.install(fusion=True)
        assert fh.get_fuser is orig
    finally:
        install_mod.uninstall()


def test_color_fuser_call_sequence(emulated, monkeypatch, tmp_path):
    """ColorFuser as get_fuser hands it out: bounds from the gt mesh, fuse_frames with .half() depth / K /
    pose and the colour frames, export_mesh writes a coloured PLY, get_mesh a trimesh with vertex colours."""
    c = make_color_tsdf_case(seed=16, frames=2, voxel_size=0.1, height=48, width=64, color_hw=(96, 128))
    corners = np.array([[c["bounds"][f"{a}min"] + 0.3, c["bounds"][f"{a}max"] - 0.3] for a in "xyz"])
    gt_mesh = types.SimpleNamespace(vertices=np.stack(np.meshgrid(*corners, indexing="ij"), -1).reshape(-1, 3))
    loads = []
    fake_trimesh = types.SimpleNamespace(Trimesh=_Recorder, load=lambda p, force=None: loads.append((p, force)) or gt_mesh)
    monkeypatch.setitem(sys.modules, "trimesh", fake_trimesh)
    cuda_calls = []
    monkeypatch.setattr(tsdf_mod.TSDF, "from_bounds", classmethod(
        lambda cls, b, voxel_size, device="cuda", color=False, _f=tsdf_mod.TSDF.from_bounds.__func__:
        cuda_calls.append(color) or _f(cls, b, voxel_size, device="cpu", color=color)))
    fuser = fusers.ColorFuser(gt_path="gt.ply", fusion_resolution=0.1, max_fusion_depth=3.0)
    assert loads == [("gt.ply", "mesh")] and cuda_calls == [True]
    tsdf = fuser.tsdf_fuser_pred.tsdf
    assert tsdf.tsdf_colors is not None and fuser.tsdf_fuser_pred.max_depth == 3.0
    fuser.fuse_frames(c["depth"], c["K"], c["cam_T_world"], c["color"])
    # what fuse_frames did, restated: the oracle on .half() inputs
    tv, tw, origin = T.new_volume({k: v for k, v in zip(c["bounds"], c["bounds"].values())}, 0.1)
    ref = tsdf_mod.TSDF.from_mesh(gt_mesh, 0.1, device="cpu", color=True)
    tv, tw, tc = ref.tsdf_values.clone(), ref.tsdf_weights.clone(), ref.tsdf_colors.clone()
    CO.integrate(tv, tw, tc, ref.origin, 0.1, c["depth"].half(), c["cam_T_world"].half(), c["K"].half(), c["color"],
                 max_depth=3.0)
    assert torch.equal(tsdf.tsdf_values, tv) and torch.equal(tsdf.tsdf_weights, tw) and torch.equal(tsdf.tsdf_colors, tc)
    fuser.export_mesh(str(tmp_path / "m.ply"))
    _, pv, pf, pc = read_ply(tmp_path / "m.ply")
    v, f, _, col = tsdf.extract_mesh(single_mesh=True, with_colors=True)
    assert len(f) > 100 and np.array_equal(pv, v.numpy()) and np.array_equal(pf, f.numpy())
    assert np.array_equal(pc, np.rint(np.float32(255) * col.numpy()).astype(np.uint8))
    _Recorder.calls.clear()
    mesh = fuser.get_mesh()
    assert _Recorder.calls == [mesh] and np.array_equal(mesh.vertex_colors, pc)
    # without colour it is OurFuser: a plain volume, colour frames ignored, a plain PLY
    plain = fusers.ColorFuser(gt_path=None, fusion_resolution=0.5, fuse_color=False)
    assert plain.tsdf_fuser_pred.tsdf.tsdf_colors is None and tuple(plain.tsdf_fuser_pred.tsdf.tsdf_values.shape) == (40, 40, 40)
