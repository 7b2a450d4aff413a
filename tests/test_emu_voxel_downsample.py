"""CPU: voxel down-sampling (csrc/srcv_voxel_downsample.cuh, DESIGN §4.19) under the host emulation (tests/emu),
through simplerecon_b200.point_cloud_fusion — points, colours and counts bitwise equal to the numpy oracle on
random, clustered, one-voxel, single-point, all-distinct, voxel-face and far-offset clouds, at sizes on both sides
of the 2048-item scan tiles and at every radix-digit count; the output order; the refusals; mesh_metrics
(down_sample=); scripts/eval_mesh.py --down-sample / --vertices; and point-cloud PLY files."""
import ctypes as C
import importlib.util
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import mesh_eval_oracle as O
from oracle import voxel_downsample_oracle as VD
from simplerecon_b200 import _native, mesh_eval as ME, point_cloud_fusion as PCF
from simplerecon_b200.tsdf import read_ply, write_ply
from tests.test_emu_mesh_eval import emulated  # noqa: F401  (the host-emulated library behind mesh_eval)


def bits(a):
    """Bit patterns, so that -0.0 and 0.0 (and NaN payloads) differ."""
    return None if a is None else np.ascontiguousarray(a).view(np.int32)


def check(points, s, colors=None):
    got = PCF.voxel_down_sample(points, s, colors)
    ref = VD.voxel_down_sample(points, s, colors)
    gp, gc, gn = (None if t is None else t.numpy() for t in got)
    assert gp.dtype == np.float32 and gn.dtype == np.int32 and gp.shape == (len(gn), 3)
    np.testing.assert_array_equal(gn, ref[2])
    np.testing.assert_array_equal(bits(gp), bits(ref[0]))
    if colors is None:
        assert gc is None
    else:
        assert gc.dtype == np.float32
        np.testing.assert_array_equal(bits(gc), bits(ref[1]))
    assert int(gn.sum()) == len(points)
    return gp, gc, gn


def u8(rng, n):
    return rng.integers(0, 256, size=(n, 3)).astype(np.uint8)


@pytest.mark.parametrize("s", [0.02, 0.03])
@pytest.mark.parametrize("color", [None, "u8", "f32", "f64"])
def test_random_cloud(emulated, s, color):
    rng = np.random.default_rng(1)
    n = 3000
    p = rng.uniform(-0.1, 0.3, size=(n, 3)).astype(np.float32)
    c = {None: None, "u8": u8(rng, n), "f32": rng.random((n, 3), dtype=np.float32),
         "f64": rng.random((n, 3))}[color]
    _, _, cnt = check(p, s, c)
    assert 1 < len(cnt) < n and cnt.max() > 1


def test_clustered_cloud(emulated):
    """Thousands of points per voxel: three tight clusters and a sparse background."""
    rng = np.random.default_rng(2)
    centres = np.array([[0.51, 0.51, 0.51], [1.03, 0.27, 0.81], [-0.4, 0.9, 0.05]])
    p = np.concatenate([c + rng.normal(scale=1e-3, size=(2500, 3)) for c in centres]
                       + [rng.uniform(-0.5, 1.1, size=(400, 3))]).astype(np.float32)
    _, _, cnt = check(p, 0.02, u8(rng, len(p)))
    assert cnt.max() >= 1000


def test_one_voxel(emulated):
    rng = np.random.default_rng(3)
    p = (np.float32(5.0) + rng.uniform(0, 0.009, size=(10_000, 3))).astype(np.float32)
    gp, gc, cnt = check(p, 0.02, rng.random((10_000, 3), dtype=np.float32))
    assert cnt.tolist() == [10_000]


def test_one_point(emulated):
    p = np.array([[-3.25, 1e4, 0.1]], np.float32)
    gp, gc, cnt = check(p, 0.02, np.array([[1, 2, 255]], np.uint8))
    np.testing.assert_array_equal(gp, p)
    assert cnt.tolist() == [1] and gc.tolist() == [[np.float32(1 / 255), np.float32(2 / 255), 1.0]]


@pytest.mark.parametrize("n", [2047, 2048, 2049, 4097])
def test_all_distinct_across_tiles(emulated, n):
    """Every point its own voxel, in shuffled order: M = N on both sides of the 2048-item tiles."""
    rng = np.random.default_rng(n)
    side = int(np.ceil(n ** (1 / 3)))
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n]
    p = (g * 0.05 + 0.01 + rng.uniform(0, 0.005, size=g.shape)).astype(np.float32)[rng.permutation(n)]
    gp, _, cnt = check(p, 0.02)
    assert len(cnt) == n and (cnt == 1).all()


@pytest.mark.parametrize("n", [2047, 2049, 6000])
def test_many_points_per_voxel_across_tiles(emulated, n):
    rng = np.random.default_rng(10 + n)
    p = rng.uniform(0, 0.1, size=(n, 3)).astype(np.float32)
    check(p, 0.03, u8(rng, n))


def test_points_on_voxel_faces_and_the_minimum(emulated):
    """Dyadic coordinates and s = 0.25: (p - b) / s is an integer for every point (b = min - s / 2), and
    the minimum point itself sits half a voxel above b."""
    rng = np.random.default_rng(4)
    k = rng.integers(0, 12, size=(1500, 3))
    p = (k * 0.25 + 0.125).astype(np.float32)         # min 0.125 -> b = 0, (p - b) / s = k + 0.5
    q = (k * 0.25).astype(np.float32)                  # min 0 -> b = -0.125, (p - b) / s = k + 0.5
    r = np.concatenate([(k * 0.25 - 0.125), [[-0.125, -0.125, -0.125]]]).astype(np.float32)
    face = np.concatenate([q, q[:1] + np.float32(0.125)])   # the minimum 0 and points on faces at k * 0.25 + 0.125
    for cloud in (p, q, r, face):
        b = cloud.astype(np.float64).min(0) - 0.125
        t = (cloud.astype(np.float64) - b) / 0.25
        assert np.array_equal(t * 2, np.round(t * 2))   # every quotient is a multiple of 1/2: on faces or centres
        check(cloud, 0.25)
        assert (VD.voxel_keys(cloud, 0.25) >= 0).all()


@pytest.mark.parametrize("offset", [-37.5, 1e4, -1e4])
def test_negative_and_far_coordinates(emulated, offset):
    rng = np.random.default_rng(5)
    p = (np.float32(offset) + rng.normal(scale=0.3, size=(2500, 3))).astype(np.float32)
    check(p, 0.02, u8(rng, len(p)))
    check(p, 0.03)


@pytest.mark.parametrize("passes", [1, 2, 3, 4, 5, 6, 7, 8])
def test_every_radix_digit_count(emulated, passes):
    """Extents whose key n_x n_y n_z - 1 needs exactly `passes` 8-bit digits."""
    rng = np.random.default_rng(20 + passes)
    bits_ = min(8 * passes, 60)                       # at most 2^20 voxels per axis here (the limit is 2^21 - 1)
    per_axis = [bits_ // 3 + (1 if a < bits_ % 3 else 0) for a in range(3)]
    ext = [1 << b for b in per_axis]                  # n_x n_y n_z = 2^bits: the top key has `bits_` bits
    s = 1.0
    v = np.stack([rng.integers(0, e, size=700) for e in ext], 1)
    v[0], v[1] = 0, np.asarray(ext) - 1               # the extent is exactly ext
    p = (v + 0.5 + rng.uniform(-0.25, 0.25, size=v.shape)).astype(np.float32)
    p[0] = 0.5                                        # the minimum: b = 0
    p = np.concatenate([p, p[rng.integers(0, len(p), 900)]])[rng.permutation(1600)]
    keys = VD.voxel_keys(p, s)
    top = int(np.prod(keys.max(0) + 1)) - 1
    assert (top.bit_length() + 7) // 8 == passes
    check(p, s, rng.random((len(p), 3)))


def test_any_input_order(emulated):
    """A permuted input: the same voxels, counts and order; each voxel's sum in the permuted order."""
    rng = np.random.default_rng(6)
    p = rng.uniform(0, 0.2, size=(3000, 3)).astype(np.float32)
    c = u8(rng, 3000)
    a = check(p, 0.02, c)
    perm = rng.permutation(3000)
    b = check(p[perm], 0.02, c[perm])
    np.testing.assert_array_equal(a[2], b[2])
    np.testing.assert_allclose(a[0], b[0], rtol=0, atol=1e-6)     # only the order of each sum differs
    k = VD.voxel_keys(p, 0.02)
    assert np.array_equal(np.unique(k, axis=0), np.unique(VD.voxel_keys(p[perm], 0.02), axis=0))


def test_deterministic(emulated):
    rng = np.random.default_rng(7)
    p = rng.uniform(0, 0.2, size=(2500, 3)).astype(np.float32)
    a = PCF.voxel_down_sample(p, 0.02)
    b = PCF.voxel_down_sample(p, 0.02)
    for x, y in zip(a[::2], b[::2]):
        assert torch.equal(x, y)


def test_refusals(emulated):
    lib = emulated
    rng = np.random.default_rng(8)
    p = rng.uniform(0, 1, size=(300, 3)).astype(np.float32)
    n0 = lib.srcv_launch_count()
    for s in (0.0, -0.02, np.nan, np.inf):
        with pytest.raises(ValueError, match="voxel_size"):
            PCF.voxel_down_sample(p, s)
    with pytest.raises(ValueError, match="empty"):
        PCF.voxel_down_sample(p[:0], 0.02)
    with pytest.raises(ValueError, match="2\\^28"):
        PCF.voxel_down_sample(torch.zeros(1, 3).expand((1 << 28) + 1, 3), 0.02)
    for c in (u8(rng, 299), np.zeros((300, 4), np.uint8), np.zeros(300, np.float32)):
        with pytest.raises(ValueError, match="colors must be \\(300, 3\\)"):
            PCF.voxel_down_sample(p, 0.02, c)
    with pytest.raises(ValueError, match="uint8, float32 or float64"):
        PCF.voxel_down_sample(p, 0.02, np.zeros((300, 3), np.int16))
    assert lib.srcv_launch_count() == n0
    bad = p.copy()
    bad[123, 1] = np.nan
    with pytest.raises(ValueError, match="voxel_down_sample: .*non-finite \\(NaN or inf\\) coordinate"):
        PCF.voxel_down_sample(bad, 0.02)
    bad[123, 1] = -np.inf
    with pytest.raises(ValueError, match="non-finite \\(NaN or inf\\) coordinate"):
        PCF.voxel_down_sample(bad, 0.02)
    c = rng.random((300, 3))
    c[7, 2] = np.inf
    with pytest.raises(ValueError, match="non-finite \\(NaN or inf\\) colour"):
        PCF.voxel_down_sample(p, 0.02, c)
    # the extent: 2^21 - 1 voxels along x passes, 2^21 raises (s = 1, b = -0.5)
    for top, ok in ((2 ** 21 - 2, True), (2 ** 21 - 1, False)):
        e = np.array([[0.0, 0.0, 0.0], [top, 0.0, 0.0], [3.0, 1.0, 2.0]], np.float32)
        assert float(e[1, 0]) == top
        if ok:
            check(e, 1.0)
        else:
            with pytest.raises(ValueError, match="2\\^21 or more voxels"):
                PCF.voxel_down_sample(e, 1.0)
            with pytest.raises(ValueError, match="2\\^21"):
                VD.voxel_down_sample(e, 1.0)
    with pytest.raises(ValueError, match="2\\^21 or more voxels"):
        PCF.voxel_down_sample(np.array([[0, 0, 0], [0, 0, 3e38]], np.float32), 1e-30)
    # the C ABI refuses what the Python layer would not pass, before any launch
    n0 = lib.srcv_launch_count()
    t = torch.zeros(64, dtype=torch.float32)
    ws = torch.empty(64, dtype=torch.uint8)
    pt = lambda x: C.c_void_p(x.data_ptr())   # noqa: E731
    assert lib.srcv_voxel_down_sample_workspace_bytes(0) == 0
    assert lib.srcv_voxel_down_sample_workspace_bytes((1 << 28) + 1) == 0
    for n, s, ct, cols, st in ((0, 0.02, 0, None, 2), ((1 << 28) + 1, 0.02, 0, None, 2), (4, 0.0, 0, None, 2),
                               (4, np.nan, 0, None, 2), (4, 0.02, 7, pt(t), 4), (4, 0.02, 1, None, 1),
                               (4, 0.02, 0, None, 3)):
        assert lib.srcv_voxel_down_sample_f32(pt(t), n, s, cols, ct, pt(t), pt(t) if cols else None, pt(t), pt(t),
                                              pt(t), pt(ws), 64, None) == st
    assert lib.srcv_launch_count() == n0


def test_mesh_metrics_down_sample_equals_oracle_sets(emulated):
    rng = np.random.default_rng(9)
    verts, faces = O.box_mesh((1.0, 0.8, 0.6))
    P = (O.sample_surface(verts, faces, 3000, seed=3) + rng.normal(scale=0.01, size=(3000, 3))).astype(np.float32)
    G = O.sample_surface(verts, faces, 3500, seed=4)
    for s in (0.02, 0.03):
        m = ME.mesh_metrics(P, G, threshold=0.02, down_sample=s)
        ref = ME.mesh_metrics(VD.voxel_down_sample(P, s)[0], VD.voxel_down_sample(G, s)[0], threshold=0.02)
        assert m == ref and m != ME.mesh_metrics(P, G, threshold=0.02)
    # a mesh side: its samples are down-sampled
    m = ME.mesh_metrics((verts, faces), G, threshold=0.02, num_samples=3000, seed=5, down_sample=0.02)
    S = ME.sample_surface(verts, faces, 3000, seed=5).numpy()
    assert m == ME.mesh_metrics(VD.voxel_down_sample(S, 0.02)[0], VD.voxel_down_sample(G, 0.02)[0], threshold=0.02)
    with pytest.raises(ValueError, match="voxel_size"):
        ME.mesh_metrics(P, G, down_sample=0.0)
    with pytest.raises(ValueError, match="2\\^21 or more voxels"):
        ME.mesh_metrics(P, G, down_sample=1e-9)


def test_eval_mesh_script_down_sample_and_vertices(emulated, tmp_path, capsys):
    spec = importlib.util.spec_from_file_location("eval_mesh", Path(__file__).resolve().parents[1] / "scripts" / "eval_mesh.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rng = np.random.default_rng(11)
    verts, faces = O.box_mesh((1.0, 0.8, 0.6))
    dense = O.sample_surface(verts, faces, 3000, seed=1)
    write_ply(tmp_path / "gt.ply", dense, rng.integers(0, 3000, size=(50, 3)))   # a mesh file: --vertices scores its vertices
    pts = (dense + rng.normal(scale=0.005, size=dense.shape)).astype(np.float32)
    write_ply(tmp_path / "pred.ply", pts, None)
    argv = [str(tmp_path / "pred.ply"), str(tmp_path / "gt.ply"), "--threshold", "0.03"]
    m = mod.main(argv + ["--down-sample", "0.02", "--vertices"])
    out = capsys.readouterr().out
    assert list(m) == list(ME.KEYS) and all(k in out for k in ME.KEYS)
    assert m == ME.mesh_metrics(pts, dense, threshold=0.03, down_sample=0.02)
    assert m["precision"] > 0.9 and m["recall"] > 0.9


def test_point_cloud_ply_round_trip(tmp_path):
    rng = np.random.default_rng(12)
    v = rng.normal(size=(50, 3)).astype(np.float32)
    c = rng.integers(0, 256, size=(50, 3)).astype(np.uint8)
    write_ply(tmp_path / "pc.ply", v, None, c)
    head = (tmp_path / "pc.ply").read_bytes().split(b"end_header\n")[0]
    assert b"element face" not in head and b"property uchar red" in head
    rv, rf = read_ply(tmp_path / "pc.ply")
    assert rf is None
    np.testing.assert_array_equal(rv, v)
    write_ply(tmp_path / "p.ply", v, None)
    rv, rf = read_ply(tmp_path / "p.ply")
    assert rf is None and np.array_equal(rv, v)
    assert len((tmp_path / "p.ply").read_bytes()) == len(
        b"ply\nformat binary_little_endian 1.0\nelement vertex 50\n"
        b"property float x\nproperty float y\nproperty float z\nend_header\n") + 50 * 12
    # with faces: the bytes the writer has always produced
    f = rng.integers(0, 50, size=(20, 3)).astype(np.int32)
    write_ply(tmp_path / "m.ply", v, f)
    data = (tmp_path / "m.ply").read_bytes()
    hdr = (b"ply\nformat binary_little_endian 1.0\nelement vertex 50\nproperty float x\nproperty float y\n"
           b"property float z\nelement face 20\nproperty list uchar int vertex_indices\nend_header\n")
    rec = np.empty(20, dtype=[("n", "u1"), ("v", "<i4", (3,))])
    rec["n"], rec["v"] = 3, f
    assert data == hdr + v.tobytes() + rec.tobytes()
