"""GPU: voxel down-sampling (DESIGN §4.19) on an H100 — bitwise equal to the numpy oracle on the CPU tier's cases
and on a process_scene cloud of more than 10^7 points, bitwise repeatable, fuse_point_cloud equal to
voxel_down_sample of process_scene's output, mesh_metrics(down_sample=) on a fused room, and device checks."""
import numpy as np
import pytest
import torch

import simplerecon_b200 as S
from oracle import mesh_eval_oracle as O
from oracle import voxel_downsample_oracle as VD
from simplerecon_b200 import point_cloud_fusion as PCF
from simplerecon_b200.synthetic import make_mvs_scene, make_tsdf_case

pytestmark = pytest.mark.gpu


def check(points, s, colors=None):
    got = PCF.voxel_down_sample(points, s, colors)
    p = points.cpu().numpy() if torch.is_tensor(points) else points
    c = colors.cpu().numpy() if torch.is_tensor(colors) else colors
    ref = VD.voxel_down_sample(p, s, c)
    gp, gc, gn = (None if t is None else t.cpu().numpy() for t in got)
    np.testing.assert_array_equal(gn, ref[2])
    np.testing.assert_array_equal(gp.view(np.int32), ref[0].view(np.int32))
    if colors is not None:
        np.testing.assert_array_equal(gc.view(np.int32), ref[1].view(np.int32))
    return got


def cases():
    rng = np.random.default_rng(0)
    u8 = lambda n: rng.integers(0, 256, size=(n, 3)).astype(np.uint8)   # noqa: E731
    yield "random", rng.uniform(-0.1, 0.3, size=(30000, 3)).astype(np.float32), 0.02, u8(30000)
    yield "random_003_f32", rng.uniform(-0.1, 0.3, size=(30000, 3)).astype(np.float32), 0.03, \
        rng.random((30000, 3), dtype=np.float32)
    cl = np.concatenate([c + rng.normal(scale=1e-3, size=(20000, 3)) for c in ((0.5, 0.5, 0.5), (1.0, 0.3, 0.8))])
    yield "clustered", cl.astype(np.float32), 0.02, u8(len(cl))
    yield "one_voxel", (5.0 + rng.uniform(0, 0.009, size=(10000, 3))).astype(np.float32), 0.02, rng.random((10000, 3))
    yield "one_point", np.array([[-3.25, 1e4, 0.1]], np.float32), 0.02, u8(1)
    g = np.stack(np.meshgrid(*[np.arange(40)] * 3, indexing="ij"), -1).reshape(-1, 3)
    yield "all_distinct", (g * 0.05 + 0.01).astype(np.float32)[rng.permutation(len(g))], 0.02, None
    k = rng.integers(0, 40, size=(20000, 3))
    yield "faces", (k * 0.25).astype(np.float32), 0.25, None
    yield "far", (np.float32(-1e4) + rng.normal(scale=2.0, size=(50000, 3))).astype(np.float32), 0.02, u8(50000)
    for n in (2047, 2048, 2049, 100_001):
        yield f"n{n}", rng.uniform(0, 0.5, size=(n, 3)).astype(np.float32), 0.02, u8(n)
    v = np.stack([rng.integers(0, 1 << 20, size=5000) for _ in range(3)], 1)
    yield "eight_passes", (v + 0.5).astype(np.float32), 1.0, None


@pytest.mark.parametrize("name,points,s,colors", list(cases()), ids=[c[0] for c in cases()])
def test_equals_oracle(cuda_device, name, points, s, colors):
    check(points, s, colors)


@pytest.fixture(scope="module")
def scene_cloud(cuda_device):
    sc = make_mvs_scene(seed=3, frames=40, height=480, width=640)
    d, E, K, im = (sc[k].to(cuda_device) for k in ("depths", "cam_T_world", "K", "images"))
    pts, rgb, _ = PCF.process_scene(d, im, E, K, 0.04, 3)
    return (d, im, E, K), pts, rgb


def test_process_scene_cloud_equals_oracle_and_repeats(cuda_device, scene_cloud):
    _, pts, rgb = scene_cloud
    assert len(pts) >= 10_000_000
    a = check(pts, 0.02, rgb)
    p = torch.from_numpy(pts).to(cuda_device)
    c = torch.from_numpy(rgb).to(cuda_device)
    b = PCF.voxel_down_sample(p, 0.02, c)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_fuse_point_cloud_equals_process_scene_then_down_sample(cuda_device, scene_cloud):
    (d, im, E, K), pts, rgb = scene_cloud
    got = S.fuse_point_cloud(d, im, E, K, z_thresh=0.04, n_consistent_thresh=3, voxel_size=0.02)
    ref = PCF.voxel_down_sample(torch.from_numpy(pts).to(cuda_device), 0.02, torch.from_numpy(rgb).to(cuda_device))
    for x, y in zip(got, ref):
        assert x.device == d.device and torch.equal(x, y)
    got_f = S.fuse_point_cloud(d[:6], im[:6].float(), E[:6], K[:6], voxel_size=0.03)
    p6, c6, _ = PCF.process_scene(d[:6], im[:6].float(), E[:6], K[:6], 0.04, 3)
    for x, y in zip(got_f, PCF.voxel_down_sample(p6, 0.03, c6)):
        assert torch.equal(x, y)


def test_mesh_metrics_down_sample_on_a_fused_room(cuda_device):
    room = (4.0, 3.0, 2.6)
    c = make_tsdf_case(seed=5, frames=12, voxel_size=0.04, height=192, width=256, room=room)
    vol = S.SparseTSDF.from_bounds(c["bounds"], 0.04, max_blocks=1 << 16)
    S.TSDFFuser(vol, max_depth=c["max_depth"]).integrate_depth(c["depth"].to(cuda_device),
                                                               c["cam_T_world"].to(cuda_device), c["K"].to(cuda_device))
    verts, faces, _ = vol.extract_mesh(single_mesh=True)
    bv, bf = (torch.from_numpy(a).to(cuda_device) for a in O.box_mesh(room))
    n = 500_000
    m = S.mesh_metrics((verts, faces), (bv, bf), threshold=0.05, num_samples=n, seed=3, down_sample=0.02)
    P = S.voxel_down_sample(S.sample_surface(verts, faces, n, seed=3), 0.02)[0]
    G = S.voxel_down_sample(S.sample_surface(bv, bf, n, seed=4), 0.02)[0]
    assert len(P) < n and len(G) < n
    assert m == S.mesh_metrics(P, G, threshold=0.05)
    assert m == S.mesh_metrics((verts, faces), (bv, bf), threshold=0.05, num_samples=n, seed=3, down_sample=0.02)


def test_devices(cuda_device):
    p = torch.rand(1000, 3, device=cuda_device)
    with pytest.raises(RuntimeError, match="CUDA"):
        PCF.voxel_down_sample(p.cpu(), 0.02)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="colors on"):
            PCF.voxel_down_sample(p, 0.02, torch.rand(1000, 3, device="cuda:1"))
    with pytest.raises((ValueError, RuntimeError)):
        PCF.voxel_down_sample(p, 0.02, torch.rand(1000, 3))
