"""CPU: the mesh-evaluation kernels (csrc/srcv_mesh_eval.cuh, DESIGN §4.17) under the host emulation (tests/emu),
through simplerecon_b200.mesh_eval — exact distances against an fp64 KD-tree on adversarial sets, exact
precision / recall counts, the sampler against the oracle's reproduction of its hash, flagged inputs, determinism,
read_ply and scripts/eval_mesh.py."""
import contextlib
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import mesh_eval_oracle as O
from simplerecon_b200 import _native, mesh_eval as ME
from simplerecon_b200.tsdf import read_ply, write_ply
from tests import emu


@pytest.fixture()
def emulated(monkeypatch):
    lib = emu.load_or_skip()
    monkeypatch.setattr(_native, "_lib", lib)
    monkeypatch.setattr(ME, "_require_cuda", lambda t: None)
    monkeypatch.setattr(ME, "_default_device", lambda: torch.device("cpu"))
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


def distances_and_stats(q, p):
    flags = torch.zeros(1, dtype=torch.int32)
    st = torch.zeros(8, dtype=torch.int64)       # per level: candidates, then queries left open
    d = ME._distances(torch.as_tensor(q).float().contiguous(), torch.as_tensor(p).float().contiguous(), flags, st)
    assert int(flags) == 0
    return d.numpy(), st.tolist()


def check_exact(q, p):
    d, st = distances_and_stats(q, p)
    ref = O.nearest_distances(q, p)
    np.testing.assert_allclose(d, ref, rtol=1e-12, atol=0)
    return st


def test_distances_planes_and_far_outliers(emulated):
    """Targets on three planes of a room corner, queries near them plus far floaters that must be queued."""
    rng = np.random.default_rng(1)
    t = rng.uniform(0, 2, size=(1500, 3))
    t[:500, 0] = 0.0
    t[500:1000, 1] = 0.0
    t[1000:, 2] = 0.0
    q = t[rng.permutation(1500)[:1200]] + rng.normal(scale=0.02, size=(1200, 3))
    mid = rng.normal(size=(40, 3)) * 20.0   # beyond the finest grid's shells: settled by a coarser level
    far = rng.normal(size=(24, 3)) * 1e5    # beyond every level: the brute-force queue
    st = check_exact(np.concatenate([q, mid, far]).astype(np.float32), t.astype(np.float32))
    assert st[0] > 0 and st[4] >= 64          # the finest level left the mid-range and far queries open
    assert 24 <= st[7] < 64                   # only the far ones reached the brute force


def test_distances_cell_faces_corners_and_duplicates(emulated):
    """128 targets on the integer lattice of [0, 8]^2 at z = 0 (duplicates included): the cell edge is
    sqrt(2 * 64 / 128) = 1, so every target lies on cell faces; queries on cell corners and centres."""
    lat = np.array([(x, y, 0) for x in range(9) for y in range(9)], np.float32)
    t = np.concatenate([lat, lat[:47]])
    assert len(t) == 128
    qs = np.array([(x, y, z) for x in range(-2, 11) for y in range(-2, 11) for z in (-1, 0, 1, 2)], np.float32)
    check_exact(np.concatenate([qs, qs[::7] + 0.5]), t)


def test_distances_single_target_and_all_equal(emulated):
    rng = np.random.default_rng(2)
    q = rng.normal(size=(300, 3)).astype(np.float32) * 5
    check_exact(q, np.array([[0.25, -1.0, 3.0]], np.float32))
    check_exact(q, np.repeat(np.array([[1.0, 2.0, 3.0]], np.float32), 40, 0))


def test_distances_clustered_targets(emulated):
    rng = np.random.default_rng(3)
    t = np.concatenate([rng.normal(size=(600, 3)) * 1e-3, rng.normal(size=(600, 3)) * 1e-3 + 30.0])
    q = np.concatenate([rng.normal(size=(400, 3)) * 1e-2, rng.normal(size=(400, 3)) * 1e-2 + 30.0,
                        rng.uniform(0, 30, size=(100, 3))])
    check_exact(q.astype(np.float32), t.astype(np.float32))


def test_sampler_matches_oracle_hash(emulated):
    """Samples equal the oracle's reproduction within 1e-6 m, except draws whose CDF value falls within rounding
    of a triangle boundary (the kernel's tiled prefix sum and np.cumsum differ in the last bits): at most 2."""
    verts, faces = O.box_mesh((4.0, 3.0, 2.6))
    verts = np.concatenate([verts, np.array([[1, 1, 1], [1.001, 1, 1], [1, 1.001, 1]], np.float32)])
    faces = np.concatenate([faces, np.array([[8, 9, 10]], np.int32)])
    for seed in (0, 12345):
        got = ME.sample_surface(torch.from_numpy(verts), torch.from_numpy(faces).long(), 5000, seed=seed).numpy()
        ref = O.sample_surface(verts, faces, 5000, seed=seed)
        off = np.abs(got - ref).max(1)
        assert np.count_nonzero(off > 1e-6) <= 2, np.sort(off)[-5:]


def test_metrics_exact_counts_and_determinism(emulated):
    rng = np.random.default_rng(4)
    verts, faces = O.box_mesh((2.0, 1.5, 1.0))
    P = O.sample_surface(verts, faces, 3000, seed=7) + rng.normal(scale=0.03, size=(3000, 3)).astype(np.float32)
    P[:20] += 3.0                           # floaters
    m1 = ME.mesh_metrics(torch.from_numpy(P), (verts, faces), threshold=0.05, num_samples=2500, seed=5)
    m2 = ME.mesh_metrics(P, (torch.from_numpy(verts), torch.from_numpy(faces)), threshold=0.05, num_samples=2500, seed=5)
    assert list(m1) == list(ME.KEYS) and m1 == m2 and all(isinstance(v, float) for v in m1.values())
    G = ME.sample_surface(verts, faces, 2500, seed=6).numpy()
    dp, dg = O.nearest_distances(P, G), O.nearest_distances(G, P)
    ref = O.metrics_from_distances(dp, dg, 0.05)
    assert m1["precision"] == np.count_nonzero(dp < 0.05) / len(P)
    assert m1["recall"] == np.count_nonzero(dg < 0.05) / len(G)
    for k in ("acc", "comp", "chamfer", "fscore"):
        assert m1[k] == pytest.approx(ref[k], rel=1e-12)
    # 2000 samples on 13 m^2: about 8 cm apart, all within 20 cm of the other side's samples
    same = ME.mesh_metrics((verts, faces), (verts, faces), threshold=0.2, num_samples=2000, seed=0)
    assert same["precision"] == same["recall"] == same["fscore"] == 1.0 and same["acc"] < 0.05


def test_flagged_inputs_give_nan_and_raise(emulated):
    verts, faces = O.box_mesh()
    pts = O.sample_surface(verts, faces, 500, seed=1)
    bad = pts.copy()
    bad[17, 1] = np.nan
    assert torch.isnan(ME.nearest_distances(bad, pts)).all()
    assert torch.isnan(ME.nearest_distances(pts, bad)).all()
    with pytest.raises(ValueError, match="non-finite"):
        ME.mesh_metrics(bad, pts)
    oor = faces.astype(np.int64).copy()
    oor[3, 2] = 8
    oor[5, 0] = 1 << 40
    assert torch.isnan(ME.sample_surface(verts, oor, 300)).all()
    with pytest.raises(ValueError, match=r"face index outside \[0, V\)"):
        ME.mesh_metrics((verts, oor), pts, num_samples=300)
    vinf = verts.copy()
    vinf[2, 0] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        ME.mesh_metrics(pts, (vinf, faces), num_samples=300)
    flat = np.zeros_like(verts)
    with pytest.raises(ValueError, match="zero total area"):
        ME.mesh_metrics((flat, faces), pts, num_samples=300)


def test_empty_inputs_refused_before_any_launch(emulated):
    lib = emulated
    n0 = lib.srcv_launch_count()
    pts = np.zeros((5, 3), np.float32)
    with pytest.raises(ValueError, match="empty"):
        ME.nearest_distances(np.zeros((0, 3), np.float32), pts)
    with pytest.raises(ValueError, match="empty"):
        ME.mesh_metrics(pts, np.zeros((0, 3), np.float32))
    with pytest.raises(ValueError, match="no faces"):
        ME.sample_surface(pts, np.zeros((0, 3), np.int64), 10)
    with pytest.raises(ValueError, match="num_samples"):
        ME.sample_surface(pts, np.array([[0, 1, 2]]), 0)
    assert lib.srcv_launch_count() == n0
    flags = torch.zeros(1, dtype=torch.int32)
    args = _native.MeshEvalArgs(0, 0, 5, flags.data_ptr(), None)
    ws = torch.empty(1024, dtype=torch.uint8)
    out = torch.empty(5, dtype=torch.float64)
    assert lib.srcv_nearest_distances_f32(C.byref(args), C.c_void_p(out.data_ptr()), C.c_void_p(out.data_ptr()),
                                          C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), 1024, None) == 2


def test_read_ply_round_trip_and_scannet_layout(tmp_path):
    rng = np.random.default_rng(5)
    v = rng.normal(size=(40, 3)).astype(np.float32)
    f = rng.integers(0, 40, size=(60, 3)).astype(np.int32)
    write_ply(tmp_path / "a.ply", v, f)
    rv, rf = read_ply(tmp_path / "a.ply")
    np.testing.assert_array_equal(rv, v)
    np.testing.assert_array_equal(rf, f)
    write_ply(tmp_path / "c.ply", v, f, rng.uniform(size=(40, 3)))
    rv, rf = read_ply(tmp_path / "c.ply")
    np.testing.assert_array_equal(rv, v)
    np.testing.assert_array_equal(rf, f)
    # ScanNet _vh_clean_2.ply: float xyz, uchar RGBA, a uchar / int face list; here with double xyz and uint indices too
    for xyz, idx in (("float", "int"), ("double", "uint")):
        hdr = ("ply\nformat binary_little_endian 1.0\ncomment VCGLIB generated\nelement vertex 40\n"
               + "".join(f"property {xyz} {a}\n" for a in "xyz")
               + "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\n"
               + f"element face 60\nproperty list uchar {idx} vertex_indices\nend_header\n")
        vt = np.empty(40, dtype=[("p", "<f8" if xyz == "double" else "<f4", (3,)), ("c", "u1", (4,))])
        vt["p"], vt["c"] = v, 200
        ft = np.empty(60, dtype=[("n", "u1"), ("v", "<u4" if idx == "uint" else "<i4", (3,))])
        ft["n"], ft["v"] = 3, f
        p = tmp_path / f"scannet_{xyz}.ply"
        p.write_bytes(hdr.encode() + vt.tobytes() + ft.tobytes())
        rv, rf = read_ply(p)
        np.testing.assert_array_equal(rv, v)
        np.testing.assert_array_equal(rf, f)
    write_ply(tmp_path / "pc.ply", v, np.zeros((0, 3), np.int32))
    assert len(read_ply(tmp_path / "pc.ply")[1]) == 0
    (tmp_path / "ascii.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nend_header\n0\n")
    with pytest.raises(ValueError, match="binary little-endian"):
        read_ply(tmp_path / "ascii.ply")


def test_eval_mesh_script(emulated, tmp_path, capsys):
    import importlib.util
    from pathlib import Path
    spec = importlib.util.spec_from_file_location("eval_mesh", Path(__file__).resolve().parents[1] / "scripts" / "eval_mesh.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    verts, faces = O.box_mesh((1.0, 1.0, 1.0))
    write_ply(tmp_path / "gt.ply", verts, faces)
    pts = O.sample_surface(verts, faces, 800, seed=9) + np.float32(0.01)
    write_ply(tmp_path / "pred.ply", pts, np.zeros((0, 3), np.int32))
    m = mod.main([str(tmp_path / "pred.ply"), str(tmp_path / "gt.ply"), "--samples", "700", "--seed", "2",
                  "--threshold", "0.25"])
    out = capsys.readouterr().out
    assert list(m) == list(ME.KEYS) and all(k in out for k in ME.KEYS)
    assert m["precision"] == 1.0 and 0.0 < m["acc"] < 0.1      # 700 samples on 6 m^2: about 9 cm apart
