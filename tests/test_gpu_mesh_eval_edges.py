"""GPU: mesh evaluation (csrc/srcv_mesh_eval.cuh, DESIGN §4.17) on an H100 at the edges where the grid search and the
sampler take their rare paths: a level-0 table whose cells collide past any probe cap, a volume-filling cloud large
enough that level 1's table overflows and is skipped, degenerate target boxes at 10^5 - 10^6 points, a brute-force
queue of 10^5 queries, and the sampler at multi-tile face counts up to about 10^6 faces.  The cases come from
tests/mesh_eval_cases.py, shared with the CPU tier.  Every distance test asserts from the search statistics
(``queued[l]``, ``candidates[l]``) which level or the brute force settled its queries.  The distance oracle is an
fp64 brute force in torch on the device, chunked over queries and targets."""
import numpy as np
import pytest
import torch

import simplerecon_b200 as S
from oracle import mesh_eval_oracle as O
from simplerecon_b200 import mesh_eval as ME
from simplerecon_b200.synthetic import make_tsdf_case
from tests import mesh_eval_cases as cases

pytestmark = pytest.mark.gpu


def brute(q: torch.Tensor, p: torch.Tensor, qchunk: int = 64, pchunk: int = 1 << 20) -> torch.Tensor:
    """Exact fp64 distances from the fp32 coordinates; at most qchunk x pchunk pairs at a time."""
    q64, p64 = q.double(), p.double()
    out = torch.empty(len(q), dtype=torch.float64, device=q.device)
    for i in range(0, len(q), qchunk):
        best = torch.full((min(qchunk, len(q) - i),), float("inf"), dtype=torch.float64, device=q.device)
        for j in range(0, len(p), pchunk):
            pj = p64[j:j + pchunk]
            d2 = (q64[i:i + qchunk, 0, None] - pj[None, :, 0]) ** 2
            for k in (1, 2):
                d2 += (q64[i:i + qchunk, k, None] - pj[None, :, k]) ** 2
            best = torch.minimum(best, d2.min(1).values)
        out[i:i + qchunk] = best.sqrt()
    return out


def distances_and_stats(q, t, dev):
    """The kernel's distances and per-level statistics: candidates evaluated [0:4], queries left open [4:8]."""
    q = torch.as_tensor(q).to(dev).float().contiguous()
    t = torch.as_tensor(t).to(dev).float().contiguous()
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    st = torch.zeros(8, dtype=torch.int64, device=dev)
    d = ME._distances(q, t, flags, st)
    assert int(flags) == 0
    return q, t, d, st.tolist()


def assert_exact(d, q, t, pick=None):
    pick = torch.arange(len(q), device=q.device) if pick is None else torch.as_tensor(pick, device=q.device)
    torch.testing.assert_close(d[pick], brute(q[pick], t), rtol=1e-12, atol=0)


def test_colliding_level0_cells_exact(cuda_device):
    t, centres, K, w = cases.colliding_level0_set(32768)
    assert K >= w + cases.MAX_PROBE
    lo, h, n = cases.level0_grid(t)
    q, t, d, st = distances_and_stats(cases.queries_near(centres, h, 2000, seed=1), t, cuda_device)
    assert_exact(d, q, t)
    assert st[0] > 0 and st[4] < len(q) // 10, st


def test_volume_cloud_level1_skipped(cuda_device):
    """The smallest power of two of uniformly filled targets at which level 1's table overflows: level 1 then
    evaluates no candidate and passes on every query level 0 left open.  One power of two lower it still searched."""
    nq = 1 << 16
    searched_below = None
    for k in range(20, 27):
        t, q, n_out = cases.volume_cloud(1 << k, nq, seed=k)
        q, t, d, st = distances_and_stats(q, t, cuda_device)
        assert st[4] >= n_out, st                     # the outside queries are beyond level 0's shells
        if st[1] == 0 and st[5] == st[4] > 0:
            break
        searched_below = st
        del q, t, d
    else:
        pytest.fail("level 1 never overflowed up to 2^26 targets")
    print(f"level 1 skipped at 2^{k} targets: stats {st}; at 2^{k - 1}: {searched_below}")
    assert searched_below is not None and searched_below[1] > 0
    assert st[7] < st[4]                              # a coarser level settled the queries level 1 passed on
    g = torch.Generator(device=cuda_device).manual_seed(k)
    pick = torch.cat([torch.randperm(n_out, generator=g, device=cuda_device)[:2000],
                      torch.randperm(nq, generator=g, device=cuda_device)[:2000]])
    assert_exact(d, q, t, pick)


def _line_case():
    t = cases.collinear(1 << 18)
    lo, h, n = cases.level0_grid(t)
    assert h == 10.0 / len(t) and (n[1:] == 1).all()               # S = 0: h = (a + b + c) / N
    rng = np.random.default_rng(1)
    near = np.zeros((3000, 3))
    near[:, 0] = rng.uniform(0, 10, 3000)
    near[:, 1:] = t[0, 1:] + rng.uniform(-h, h, (3000, 2))
    far = near[:1000] + [0.0, 0.5, 0.0]                             # beyond every level's shells: brute force
    return t, np.concatenate([near, far]), 1000


def _plane_case():
    t = cases.coplanar(1 << 18)
    lo, h, n = cases.level0_grid(t)
    assert n[2] == 1 and n[0] > 100
    rng = np.random.default_rng(2)
    near = np.stack([rng.uniform(0, 4, 3000), rng.uniform(0, 3, 3000), 0.5 + rng.uniform(-h, h, 3000)], 1)
    mid = near[:1000] + [0.0, 0.0, 1.0]                             # past levels 0 and 1, within level 2's
    return t, np.concatenate([near, mid]), 1000


def _clusters_case():
    t = cases.far_clusters(1 << 19)
    lo, h, n = cases.level0_grid(t)
    e = t.astype(np.float64).max(0) - t.astype(np.float64).min(0)
    assert h == e.max() / (cases.KEY_BIAS - 2) and n[0] == cases.KEY_BIAS - 1   # the 2^20-cells cap binds
    rng = np.random.default_rng(3)
    near = t[rng.integers(0, len(t), 3000)] + rng.uniform(-1e-3, 1e-3, (3000, 3))
    mid = np.stack([rng.uniform(400, 600, 1000), rng.uniform(-1, 1, 1000), rng.uniform(-1, 1, 1000)], 1)
    return t, np.concatenate([near, mid]), 1000


def _equal_case():
    t = cases.all_equal(100_000)
    rng = np.random.default_rng(4)
    near = t[0] + rng.uniform(-3, 3, (3000, 3))                     # one cell (h = 1): covered within 3 shells
    far = t[0] + rng.normal(size=(1000, 3)) * 1e4
    far[np.abs(far - t[0]).max(1) < 4000, 0] = t[0, 0] + 5000.0      # beyond level 3's 5 cells of 512
    return t, np.concatenate([near, far]), 1000


def _lattice_case():
    t, q = cases.lattice(301)
    assert cases.level0_grid(t)[1] == 1.0
    return t, q, 0


@pytest.mark.parametrize("case", ["line", "plane", "clusters", "equal", "lattice"])
def test_degenerate_targets(cuda_device, case):
    """Near queries settle at level 0; the last ``n_out`` queries are placed where level 0 cannot settle them:
    for the line, the clusters and the single point beyond every level (the brute force takes exactly them),
    for the plane past levels 0 and 1 but within level 2's shells."""
    t, q, n_out = {"line": _line_case, "plane": _plane_case, "clusters": _clusters_case, "equal": _equal_case,
                   "lattice": _lattice_case}[case]()
    q, t, d, st = distances_and_stats(q.astype(np.float32), t, cuda_device)
    assert st[0] > 0, st
    if case == "line":              # a gap of 4 cells around a near query is rare, of 32 never
        assert n_out <= st[4] <= n_out + 30 and st[5] == st[7] == n_out, st
    elif case == "plane":
        assert st[4] == st[5] == n_out and st[2] > 0 and st[7] == 0, st
    else:
        assert st[4] == st[7] == n_out, st
    g = torch.Generator(device=cuda_device).manual_seed(5)
    pick = torch.randperm(len(q) - n_out, generator=g, device=cuda_device)[:20000]
    assert_exact(d, q, t, torch.cat([pick, torch.arange(len(q) - n_out, len(q), device=cuda_device)]))


def test_brute_force_queue_of_1e5(cuda_device):
    """10^5 queries 10 km from 10^5 targets: every level passes them on, and the brute force covers
    ceil(10^5 / 256) x ceil(10^5 / 8192) = 391 x 13 work items."""
    rng = np.random.default_rng(6)
    t = rng.random((100_000, 3), dtype=np.float32)
    q = rng.normal(size=(100_000, 3))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True) * rng.uniform(1e4, 2e4, (100_000, 1))).astype(np.float32)
    q, t, d, st = distances_and_stats(q, t, cuda_device)
    assert st[4:] == [len(q)] * 4 and st[:4] == [0, 0, 0, 0], st
    assert_exact(d, q, t)


def _room_mesh(dev):
    """The fused synthetic room at 1.6 cm: about 10^6 faces."""
    room = (6.0, 5.0, 3.0)
    vol = S.SparseTSDF(0.016, max_blocks=1 << 17)
    fuser = S.TSDFFuser(vol, max_depth=3.0)
    for i in range(4):
        c = make_tsdf_case(seed=200 + i, frames=8, voxel_size=0.016, height=240, width=320, room=room)
        fuser.integrate_depth(c["depth"].to(dev), c["cam_T_world"].to(dev), c["K"].to(dev))
    verts, faces, _ = vol.extract_mesh(single_mesh=True)
    return verts.float().cpu().numpy(), faces.int().cpu().numpy()


@pytest.mark.parametrize("name", [*cases.SAMPLER_MESHES, cases.LARGE_SAMPLER_MESH, "fused_room"])
def test_sampler_across_scan_tiles(cuda_device, name):
    """10^6 samples: per-face counts within 2 of N A_f / A (zero-area faces none), and every sample the oracle's
    or, for a draw within rounding of a CDF boundary, the oracle's point on the neighbouring triangle."""
    if name == "fused_room":
        verts, faces = _room_mesh(cuda_device)
        assert len(faces) > 800_000
    else:
        verts, faces = cases.sampler_mesh(name)
    N, seed = 1_000_000, 9
    got = S.sample_surface(torch.from_numpy(verts).to(cuda_device), torch.from_numpy(faces).to(cuda_device), N,
                           seed=seed).cpu().numpy()
    areas = cases.triangle_areas(verts, faces)
    face, moved = cases.check_against_oracle(got, verts, faces, N, seed, O)
    if name != "fused_room":
        np.testing.assert_array_equal(face, cases.strip_faces_of(got, verts, faces))
    cases.check_stratified_counts(face, areas, N)
    print(f"{name}: {len(faces)} faces, {moved} samples on a neighbouring triangle")
