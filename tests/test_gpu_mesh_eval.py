"""GPU: mesh evaluation (DESIGN §4.17) on an H100 — exact nearest distances at 10^6 x 10^6 with far outliers, the
metrics of the fused synthetic room (dense TSDF and SparseTSDF) against the analytic box, bitwise determinism, and
no host synchronisation in sample_surface / nearest_distances.  The distance oracle is a chunked fp64 brute force
in torch on the device."""
import pytest
import torch

import simplerecon_b200 as S
from oracle import mesh_eval_oracle as O
from simplerecon_b200.synthetic import make_tsdf_case

pytestmark = pytest.mark.gpu


def brute(q: torch.Tensor, p: torch.Tensor, chunk: int = 128) -> torch.Tensor:
    """Exact fp64 distances from the fp32 coordinates, chunk queries at a time."""
    q64, p64 = q.double(), p.double()
    out = torch.empty(len(q), dtype=torch.float64, device=q.device)
    for i in range(0, len(q), chunk):
        d2 = torch.zeros(min(chunk, len(q) - i), len(p), dtype=torch.float64, device=q.device)
        for k in range(3):
            d2 += (q64[i:i + chunk, k, None] - p64[None, :, k]) ** 2
        out[i:i + chunk] = d2.min(1).values.sqrt()
    return out


def test_nearest_distances_million_with_far_outliers(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(0)
    n = 1_000_000
    verts, faces = O.box_mesh((6.0, 5.0, 3.0))
    p = S.sample_surface(torch.from_numpy(verts).to(cuda_device), torch.from_numpy(faces).to(cuda_device), n, seed=1)
    q = S.sample_surface(torch.from_numpy(verts).to(cuda_device), torch.from_numpy(faces).to(cuda_device), n, seed=2)
    q = q + 0.02 * torch.randn(q.shape, generator=g, device=cuda_device)
    far = torch.randperm(n, generator=g, device=cuda_device)[: n // 100]
    q[far] = q[far] + 50.0 * torch.randn(len(far), 3, generator=g, device=cuda_device)
    d = S.nearest_distances(q, p)
    assert d.dtype == torch.float64 and d.shape == (n,)
    pick = torch.cat([far[:3000], torch.randperm(n, generator=g, device=cuda_device)[:5000]])
    ref = brute(q[pick], p)
    torch.testing.assert_close(d[pick], ref, rtol=1e-12, atol=0)


@pytest.mark.parametrize("sparse", [False, True])
def test_fused_room_against_the_box(cuda_device, sparse):
    voxel = 0.04
    c = make_tsdf_case(seed=5, frames=12, voxel_size=voxel, height=192, width=256)
    vol = (S.SparseTSDF.from_bounds(c["bounds"], voxel, max_blocks=1 << 16) if sparse
           else S.TSDF.from_bounds(c["bounds"], voxel))
    S.TSDFFuser(vol, max_depth=c["max_depth"]).integrate_depth(c["depth"].to(cuda_device), c["cam_T_world"].to(cuda_device),
                                                               c["K"].to(cuda_device))
    verts, faces, _ = vol.extract_mesh(single_mesh=True)
    assert len(faces) > 10000
    bv, bf = (torch.from_numpy(a).to(cuda_device) for a in O.box_mesh((4.0, 3.0, 2.6)))
    n = 100_000
    m = S.mesh_metrics((verts, faces), (bv, bf), threshold=0.05, num_samples=n, seed=3)
    P = S.sample_surface(verts, faces, n, seed=3)
    G = S.sample_surface(bv, bf, n, seed=4)
    dp, dg = brute(P, G), brute(G, P)
    assert m["precision"] == int((dp < 0.05).sum()) / n and m["recall"] == int((dg < 0.05).sum()) / n
    ref = O.metrics_from_distances(dp.cpu().numpy(), dg.cpu().numpy(), 0.05)
    for k in ("acc", "comp", "chamfer", "fscore"):
        assert m[k] == pytest.approx(ref[k], rel=1e-12)
    assert m["acc"] < voxel
    assert m == S.mesh_metrics((verts, faces), (bv, bf), threshold=0.05, num_samples=n, seed=3)


def test_same_seed_bitwise_and_no_host_sync(cuda_device):
    bv, bf = (torch.from_numpy(a).to(cuda_device) for a in O.box_mesh((4.0, 3.0, 2.6)))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = S.sample_surface(bv, bf, 300_000, seed=11)
        b = S.sample_surface(bv, bf, 300_000, seed=11)
        d1 = S.nearest_distances(a, b[::3])
        d2 = S.nearest_distances(a, b[::3].contiguous())
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(a, b) and torch.equal(d1, d2)
    m1 = S.mesh_metrics(a, (bv, bf), num_samples=300_000, seed=7)
    m2 = S.mesh_metrics(a, (bv, bf), num_samples=300_000, seed=7)
    assert m1 == m2
