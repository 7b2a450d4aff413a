"""GPU: visibility culling of mesh evaluation (DESIGN §4.18) on an H100 — observation counts equal to the oracle at
10^6 points x 64 frames, the fused SparseTSDF room against the box with its own fusion frames as views (metrics
against scipy's cKDTree on the oracle-culled sample sets, bitwise repeatable), and no host synchronisation in
observation_counts."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import simplerecon_b200 as S
from oracle import mesh_eval_oracle as O
from oracle import mesh_visibility_oracle as VO
from simplerecon_b200.synthetic import make_tsdf_case

pytestmark = pytest.mark.gpu

ROOM = (4.0, 3.0, 2.6)


def test_counts_equal_oracle_million_points_64_frames(cuda_device):
    c = make_tsdf_case(seed=9, frames=64, height=240, width=320, room=ROOM)
    d = c["depth"].clone()
    d[torch.rand(d.shape, generator=torch.Generator().manual_seed(1)) < 0.05] = float("nan")
    d, K, E = d.to(cuda_device), c["K"].to(cuda_device), c["cam_T_world"].to(cuda_device)
    bv, bf = (torch.from_numpy(a).to(cuda_device) for a in O.box_mesh(ROOM))
    n = 1_000_000
    surf = S.sample_surface(bv, bf, n - n // 10, seed=1)
    g = torch.Generator(device=cuda_device).manual_seed(2)
    rest = (torch.rand(n // 10, 3, generator=g, device=cuda_device) * 6.0 - 1.0) * torch.tensor(ROOM, device=cuda_device)
    p = torch.cat([surf, rest])
    got = S.observation_counts(p, d, K, E, max_depth=3.0)
    ref = VO.observation_counts_torch(p, d, K, E, max_depth=3.0)
    assert got.dtype == torch.int32 and torch.equal(got, ref)
    pick = torch.randperm(n, generator=g, device=cuda_device)[:20000].cpu().numpy()
    np.testing.assert_array_equal(got.cpu().numpy()[pick],
                                  VO.observation_counts(p.cpu().numpy()[pick], d.cpu().numpy(), K.cpu().numpy(),
                                                        E.cpu().numpy(), max_depth=3.0))
    assert 0.2 < float((got > 0).float().mean()) < 0.95


@pytest.fixture(scope="module")
def fused_room(cuda_device):
    c = make_tsdf_case(seed=5, frames=12, voxel_size=0.04, height=192, width=256, room=ROOM)
    vol = S.SparseTSDF.from_bounds(c["bounds"], 0.04, max_blocks=1 << 16)
    d, E, K = c["depth"].to(cuda_device), c["cam_T_world"].to(cuda_device), c["K"].to(cuda_device)
    S.TSDFFuser(vol, max_depth=c["max_depth"]).integrate_depth(d, E, K)
    verts, faces, _ = vol.extract_mesh(single_mesh=True)
    return (verts, faces), S.Views(d, K, E, margin=0.05, max_depth=c["max_depth"])


def test_fused_room_culled_metrics_against_ckdtree(cuda_device, fused_room):
    (verts, faces), views = fused_room
    bv, bf = (torch.from_numpy(a).to(cuda_device) for a in O.box_mesh(ROOM))
    n = 200_000
    m = S.mesh_metrics((verts, faces), (bv, bf), threshold=0.05, num_samples=n, seed=3, views=views)
    P = S.sample_surface(verts, faces, n, seed=3).cpu().numpy()
    G = S.sample_surface(bv, bf, n, seed=4).cpu().numpy()
    d, K, E = (t.cpu().numpy() for t in views[:3])
    Pk = P[VO.observation_counts(P, d, K, E, views.margin, views.max_depth) > 0]
    Gk = G[VO.observation_counts(G, d, K, E, views.margin, views.max_depth) > 0]
    assert 0 < len(Gk) < n and 0 < len(Pk) <= n
    dp = cKDTree(Gk.astype(np.float64)).query(Pk.astype(np.float64), k=1, workers=-1)[0]
    dg = cKDTree(Pk.astype(np.float64)).query(Gk.astype(np.float64), k=1, workers=-1)[0]
    assert m["precision"] == np.count_nonzero(dp < 0.05) / len(Pk)
    assert m["recall"] == np.count_nonzero(dg < 0.05) / len(Gk)
    ref = O.metrics_from_distances(dp, dg, 0.05)
    for k in ("acc", "comp", "chamfer", "fscore"):
        assert m[k] == pytest.approx(ref[k], rel=1e-12)
    assert m == S.mesh_metrics((verts, faces), (bv, bf), threshold=0.05, num_samples=n, seed=3, views=views)
    full = S.mesh_metrics((verts, faces), (bv, bf), threshold=0.05, num_samples=n, seed=3)
    assert m["recall"] > full["recall"]                  # walls the frames never saw no longer count as missed


def test_observation_counts_bitwise_and_no_host_sync(cuda_device, fused_room):
    (verts, faces), views = fused_room
    p = S.sample_surface(verts, faces, 300_000, seed=11)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = S.observation_counts(p, *views)
        b = S.observation_counts(p, views.depths[:5], views.K[:5], views.cam_T_world[:5], views.margin, views.max_depth)
        b = S.observation_counts(p, views.depths[5:], views.K[0], views.cam_T_world[5:], views.margin, views.max_depth,
                                 counts=b)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(a, b) and int((a > 0).sum()) > 0.9 * len(p)
