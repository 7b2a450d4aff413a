"""CPU: visibility culling of mesh evaluation (csrc/srcv_mesh_visibility.cuh, DESIGN §4.18) under the host emulation
(tests/emu), through simplerecon_b200.mesh_eval — observation counts equal to the numpy oracle exactly (noisy room
views with holes, constructed pixel / depth / margin boundaries, any point order, chunked frames), an analytic box
room, culled metrics against the oracle, flagged and refused inputs, scripts/eval_mesh.py --views, and what ptxas
makes of the kernels."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import mesh_eval_oracle as O
from oracle import mesh_visibility_oracle as VO
from simplerecon_b200 import _native, build as B, mesh_eval as ME
from simplerecon_b200.synthetic import make_tsdf_case
from simplerecon_b200.tsdf import write_ply
from tests.test_emu_mesh_eval import emulated  # noqa: F401  (the host-emulated library behind mesh_eval)

ROOM = (4.0, 3.0, 2.6)


def counts_of(points, depths, K, E, **kw):
    return ME.observation_counts(points, depths, K, E, **kw).numpy()


def room_views(frames=6, holes=None, seed=3):
    c = make_tsdf_case(seed=seed, frames=frames, height=48, width=64, room=ROOM)
    d = c["depth"][:, 0].numpy().copy()
    if holes is not None:
        rng = np.random.default_rng(seed)
        d[rng.random(d.shape) < 0.15] = holes
    return d, c["K"].numpy(), c["cam_T_world"].numpy()


def room_points(n=4000, seed=0):
    """Box samples (triangle order), points inside the room and far outside it."""
    rng = np.random.default_rng(seed)
    verts, faces = O.box_mesh(ROOM)
    surf = O.sample_surface(verts, faces, n, seed=seed)
    inside = rng.uniform(-0.2, 1.0, size=(n // 4, 3)) * ROOM
    far = rng.normal(size=(n // 8, 3)) * 100.0
    return np.concatenate([surf, inside, far]).astype(np.float32)


@pytest.mark.parametrize("holes", [None, 0.0, np.nan])
@pytest.mark.parametrize("max_depth", [np.inf, 3.0])
def test_counts_equal_oracle_on_room_views(emulated, holes, max_depth):
    d, K, E = room_views(holes=holes)
    p = room_points()
    got = counts_of(p, d[:, None], K, E, max_depth=max_depth)
    ref = VO.observation_counts(p, d, K, E, max_depth=max_depth)
    assert got.dtype == np.int32 and got.shape == (len(p),)
    np.testing.assert_array_equal(got, ref)
    assert 0 < np.count_nonzero(got) < len(p) and got.max() >= 2


def test_constructed_boundaries(emulated):
    """Dyadic K and E and power-of-two depths: u, v, z, d - z land exactly on the rule's edges."""
    H, W = 4, 8
    K = np.eye(4, dtype=np.float32)
    K[0, 0], K[0, 2], K[1, 1], K[1, 2] = 2.0, 4.0, 2.0, 2.0      # u = 2 x / z + 4, v = 2 y / z + 2
    E = np.eye(4, dtype=np.float32)[None]
    depth = np.full((1, H, W), 2.0, np.float32)
    depth[0, :, 3] = 0.0                                         # a hole in column 3
    depth[0, 0, 6] = 4.0                                         # d = max_depth
    pts, expect = [], []

    def at(u, v, z, observed):
        pts.append(((u - 4.0) * z / 2.0, (v - 2.0) * z / 2.0, z))
        expect.append(observed)

    for u, obs in ((0.0, 1), (-0.5, 0), (0.5, 1), (1.0, 1), (7.0, 1), (7.5, 1), (8.0, 0), (8.5, 0),
                   (3.0, 1),      # u - 0.5 = 2.5 rounds to 2 (half to even), not into the hole at 3
                   (4.0, 1),      # 3.5 rounds to 4, not into the hole
                   (3.25, 0), (3.5, 0)):                         # 2.75 and 3.0 hit column 3
        at(u, 2.25, 2.0, obs)
    for v, obs in ((0.0, 1), (-0.5, 0), (4.0, 0), (3.5, 1), (3.75, 1)):
        at(5.25, v, 2.0, obs)
    at(6.25, 0.25, 2.0, 0)                                       # its depth is max_depth
    at(5.25, 2.25, 0.0, 0)                                       # z = 0
    at(5.25, 2.25, -1.0, 0)                                      # behind the camera
    at(5.25, 2.25, 4.0, 0)                                       # z = max_depth
    at(5.25, 2.25, 2.25, 0)                                      # d - z = -margin exactly
    at(5.25, 2.25, 2.125, 1)                                     # d - z = -margin / 2
    p = np.asarray(pts, np.float32)
    assert np.array_equal(p.astype(np.float64), np.asarray(pts))  # every coordinate is exact in fp32
    for max_depth, margin in ((4.0, 0.25), (np.inf, 0.25)):
        got = counts_of(p, depth, K[None].repeat(1, 0), E, margin=margin, max_depth=max_depth)
        np.testing.assert_array_equal(got, VO.observation_counts(p, depth, K, E, margin=margin, max_depth=max_depth))
        if max_depth == 4.0:
            np.testing.assert_array_equal(got, expect)
    # once max_depth is inf the pixel of depth 4 counts
    got = counts_of(p, depth, K, E, margin=0.25)
    assert got[len(expect) - 6] == 1 and expect[len(expect) - 6] == 0


def test_any_point_order_gives_the_same_counts(emulated):
    d, K, E = room_views()
    p = room_points()
    perm = np.random.default_rng(1).permutation(len(p))
    st_sorted, st_random, st_all = (torch.zeros(1, dtype=torch.int64) for _ in range(3))
    a = ME._observation_counts(p, d, K, E, stats=st_sorted).numpy()
    b = ME._observation_counts(p[perm], d, K, E, stats=st_random).numpy()
    c = ME._observation_counts(p, d, K, E, tile_cull=False, stats=st_all).numpy()
    np.testing.assert_array_equal(a[perm], b)
    np.testing.assert_array_equal(a, c)
    assert int(st_all) == len(p) * len(d)                        # without the tile test every pair is evaluated
    assert int(st_sorted) < int(st_random) <= int(st_all)        # the sampler's coherent order culls the most


def test_chunked_frames_and_shared_K(emulated):
    d, K, E = room_views()
    p = room_points()
    one = counts_of(p, d, K, E)
    acc = ME.observation_counts(p, d[:2], K[:2], E[:2])
    out = ME.observation_counts(p, d[2:], K[2:], E[2:], counts=acc)
    assert out is acc
    np.testing.assert_array_equal(acc.numpy(), one)
    assert np.array_equal(K, np.broadcast_to(K[0], K.shape))
    np.testing.assert_array_equal(counts_of(p, d, K[0], E), one)


def raycast_box(K, E, H, W, room):
    """Noise-free depth (z) of the box room [0, room] seen from inside by camera E (world -> camera)."""
    R, t = E[:3, :3].astype(np.float64), E[:3, 3].astype(np.float64)
    c = -R.T @ t
    v, u = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
    rays = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1) @ R   # z = 1
    with np.errstate(divide="ignore"):
        tt = np.where(rays > 0, (np.asarray(room) - c) / rays, -c / rays)
    return tt.min(-1).astype(np.float32)


def test_analytic_box_room_one_camera(emulated):
    """A camera at the centre of the room facing the +x wall, whose frustum lies inside that wall: the observed box
    samples are exactly that wall's samples inside the image, and none behind the camera."""
    H, W = 48, 64
    K = np.eye(4, dtype=np.float32)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = 57.0, 57.0, 32.0, 24.0
    centre = np.array(ROOM) / 2
    R = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], np.float64)  # camera z = world x, camera x = -world y
    E = np.eye(4, dtype=np.float32)
    E[:3, :3], E[:3, 3] = R, -R @ centre
    depth = raycast_box(K, E, H, W, ROOM)
    assert np.allclose(depth, ROOM[0] - centre[0])               # the whole image sees the far wall
    verts, faces = O.box_mesh(ROOM)
    s = ME.sample_surface(verts, faces, 20000, seed=5).numpy()
    got = counts_of(s, depth[None], K, E[None]) > 0
    cam = (s.astype(np.float64) - centre) @ R.T
    u, v = K[0, 0] * cam[:, 0] / cam[:, 2] + K[0, 2], K[1, 1] * cam[:, 1] / cam[:, 2] + K[1, 2]
    far = s[:, 0] == np.float32(ROOM[0])
    inside = far & (u >= 0) & (u < W) & (v >= 0) & (v < H)
    edge = far & ((np.minimum(np.abs(u), np.abs(u - W)) < 1e-6) | (np.minimum(np.abs(v), np.abs(v - H)) < 1e-6))
    np.testing.assert_array_equal(got[~edge], inside[~edge])
    assert inside.sum() > 500 and not got[cam[:, 2] <= 0].any()


def test_culled_metrics_equal_oracle(emulated):
    d, K, E = room_views()
    verts, faces = O.box_mesh(ROOM)
    pv, pf = O.box_mesh((3.9, 2.95, 2.5), origin=(0.05, 0.0, 0.04))
    views = ME.Views(d[:, None], K, E)
    m = ME.mesh_metrics((pv, pf), (verts, faces), threshold=0.05, num_samples=3000, seed=2, views=views)
    m2 = ME.mesh_metrics((pv, pf), (verts, faces), threshold=0.05, num_samples=3000, seed=2, views=tuple(views))
    assert m == m2 and list(m) == list(ME.KEYS)
    P = ME.sample_surface(pv, pf, 3000, seed=2).numpy()
    G = ME.sample_surface(verts, faces, 3000, seed=3).numpy()
    Pk, Gk = P[VO.observation_counts(P, d, K, E) > 0], G[VO.observation_counts(G, d, K, E) > 0]
    assert 0 < len(Gk) < len(G) and 0 < len(Pk) < len(P)
    dp, dg = O.nearest_distances(Pk, Gk), O.nearest_distances(Gk, Pk)
    assert m["precision"] == np.count_nonzero(dp < 0.05) / len(Pk)
    assert m["recall"] == np.count_nonzero(dg < 0.05) / len(Gk)
    ref = O.metrics_from_distances(dp, dg, 0.05)
    for k in ("acc", "comp", "chamfer", "fscore"):
        assert m[k] == pytest.approx(ref[k], rel=1e-12)


def test_flags_raise(emulated):
    d, K, E = room_views()
    views = ME.Views(d, K, E)
    verts, faces = O.box_mesh(ROOM)
    pts = O.sample_surface(verts, faces, 2000, seed=1)
    bad = pts.copy()
    bad[5, 2] = np.nan
    with pytest.raises(ValueError, match="non-finite \\(NaN or inf\\) coordinate"):
        ME.mesh_metrics(bad, pts, views=views)
    Ebad = E.copy()
    Ebad[2, 1, 3] = np.inf
    with pytest.raises(ValueError, match="non-finite entry in a view"):
        ME.mesh_metrics(pts, pts, views=ME.Views(d, K, Ebad))
    Kbad = K.copy()
    Kbad[0, 0, 0] = np.nan
    with pytest.raises(ValueError, match="non-finite entry in a view"):
        ME.mesh_metrics(pts, pts, views=ME.Views(d, Kbad, E))
    with pytest.raises(ValueError, match="no point of gt"):
        ME.mesh_metrics(pts, pts + np.float32(100.0), views=views)
    with pytest.raises(ValueError, match="no point of pred"):
        ME.mesh_metrics(pts - np.float32(100.0), pts, views=views)
    # a NaN point raises also in a tile of points far outside the room, which the frustum test culls
    away = np.concatenate([pts, np.full((256, 3), -1e3, np.float32)])
    away[-7] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        ME.mesh_metrics(away, pts, views=views)


def test_bad_shapes_refused_before_any_launch(emulated):
    lib = emulated
    d, K, E = room_views()
    p = room_points(400)
    n0 = lib.srcv_launch_count()
    for args, kw, what in (((p, d[0], K, E), {}, "depths"), ((p, d, K[:, :3, :3], E), {}, "K"),
                           ((p, d, K, E[:4]), {}, "cam_T_world"), ((p, d, K[:5], E), {}, "K"),
                           ((p, d, K, E), {"margin": -0.1}, "margin"), ((p, d, K, E), {"margin": np.nan}, "margin"),
                           ((p, d, K, E), {"max_depth": 0.0}, "max_depth"),
                           ((p, d, K, E), {"counts": torch.zeros(len(p), dtype=torch.int64)}, "counts"),
                           ((p, d, K, E), {"counts": torch.zeros(len(p) - 1, dtype=torch.int32)}, "counts"),
                           ((p[:0], d, K, E), {}, "empty"), ((p, d[:0], K[:0], E[:0]), {}, "depths")):
        with pytest.raises(ValueError, match=what):
            ME.observation_counts(*args, **kw)
    with pytest.raises(TypeError):
        ME.mesh_metrics(p, p, views=(d,))
    assert lib.srcv_launch_count() == n0
    # the C ABI refuses what the Python layer would not pass
    t = torch.zeros(64, dtype=torch.float32)
    flags = torch.zeros(1, dtype=torch.int32)
    args = _native.MeshEvalArgs(0, 0, 4, flags.data_ptr(), None)
    for F, H, W, margin, max_depth in ((0, 4, 4, 0.05, 1.0), (1, 1 << 16, 1 << 15, 0.05, 1.0), (1, 4, 4, np.inf, 1.0),
                                       (1, 4, 4, 0.05, np.nan), (1, 0, 4, 0.05, 1.0)):
        v = _native.MeshViews(t.data_ptr(), t.data_ptr(), t.data_ptr(), F, H, W, 0, margin, max_depth, 1)
        assert lib.srcv_observation_counts_f32(C.byref(args), C.byref(v), C.c_void_p(t.data_ptr()),
                                               C.c_void_p(t.data_ptr()), None) == 2
    v = _native.MeshViews(t.data_ptr(), t.data_ptr(), t.data_ptr(), 1, 4, 4, 0, 0.05, 1.0, 1)
    args0 = _native.MeshEvalArgs(0, 0, 0, flags.data_ptr(), None)
    assert lib.srcv_observation_counts_f32(C.byref(args0), C.byref(v), C.c_void_p(t.data_ptr()),
                                           C.c_void_p(t.data_ptr()), None) == 2
    ws = torch.empty(8, dtype=torch.uint8)
    assert lib.srcv_compact_observed_f32(C.byref(args), C.c_void_p(t.data_ptr()), C.c_void_p(t.data_ptr()),
                                         C.c_void_p(t.data_ptr()), C.c_void_p(t.data_ptr()), C.c_void_p(ws.data_ptr()),
                                         8, None) == 3
    assert lib.srcv_launch_count() == n0


def test_compaction_keeps_input_order(emulated):
    rng = np.random.default_rng(7)
    n = 5000                                                     # three scan tiles
    p = rng.normal(size=(n, 3)).astype(np.float32)
    counts = torch.from_numpy(rng.integers(0, 3, n).astype(np.int32) * (rng.random(n) < 0.3))
    flags = torch.zeros(1, dtype=torch.int32)
    num = torch.zeros(1, dtype=torch.int64)
    out = ME._compact(torch.from_numpy(p), counts, flags, num)
    k = int(num)
    assert k == int((counts > 0).sum())
    np.testing.assert_array_equal(out[:k].numpy(), p[counts.numpy() > 0])


def test_eval_mesh_script_with_views(emulated, tmp_path, capsys):
    import importlib.util
    from pathlib import Path
    spec = importlib.util.spec_from_file_location("eval_mesh", Path(__file__).resolve().parents[1] / "scripts" / "eval_mesh.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    d, K, E = room_views()
    np.savez(tmp_path / "views.npz", depths=d, K=K[0], cam_T_world=E)
    verts, faces = O.box_mesh(ROOM)
    write_ply(tmp_path / "gt.ply", verts, faces)
    pts = O.sample_surface(verts, faces, 1500, seed=9) + np.float32(0.01)
    write_ply(tmp_path / "pred.ply", pts, np.zeros((0, 3), np.int32))
    argv = [str(tmp_path / "pred.ply"), str(tmp_path / "gt.ply"), "--samples", "1200", "--threshold", "0.25"]
    m = mod.main(argv + ["--views", str(tmp_path / "views.npz"), "--margin", "0.1", "--max-depth", "3"])
    out = capsys.readouterr().out
    assert list(m) == list(ME.KEYS) and all(k in out for k in ME.KEYS)
    assert m["precision"] > 0.9 and m["recall"] > 0.9
    assert m == ME.mesh_metrics(pts, (verts, faces), threshold=0.25, num_samples=1200,
                                views=ME.Views(d, K[0], E, margin=0.1, max_depth=3.0))


VISIBILITY_KERNELS = ("observation_count_kernel", "keep_kernel", "compact_kernel")


@pytest.fixture(scope="module")
def ptxas_props(tmp_path_factory) -> dict:
    try:
        nvcc = B.nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    flags = [f for f in B.NVCC_FLAGS if f != "-shared"]
    out = tmp_path_factory.mktemp("ptxas") / "srcv_tsdf.cubin"
    r = subprocess.run([nvcc, *flags, *B.NVCC_DEFINES, "-Xptxas", "-v", "-cubin", "-o", str(out),
                        str(B.PKG / "csrc" / "srcv_tsdf.cu")], capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed:\n{r.stderr[-4000:]}"
    return {name: (int(stack), int(st), int(ld)) for name, stack, st, ld in re.findall(
        r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
        r.stdout + r.stderr)}


@pytest.mark.parametrize("kernel", VISIBILITY_KERNELS)
def test_visibility_kernels_no_spills_no_stack(ptxas_props, kernel):
    hits = {k: v for k, v in ptxas_props.items() if "mesh_vis_detail" in k and kernel in k}
    assert hits, f"no {kernel} in the ptxas output"
    for name, props in hits.items():
        assert props == (0, 0, 0), f"{name}: stack {props[0]}, spill stores {props[1]}, spill loads {props[2]}"
