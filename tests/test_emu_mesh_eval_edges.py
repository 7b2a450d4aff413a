"""CPU: the mesh-evaluation kernels (csrc/srcv_mesh_eval.cuh, DESIGN §4.17) under the host emulation at the edges the
everyday cases miss — a level-0 hash table whose cells collide past any probe cap, and the sampler's prefix sum
across several scan tiles — against the numpy oracle (oracle/mesh_eval_oracle.py).  The cases come from
tests/mesh_eval_cases.py, which the GPU tier shares."""
import numpy as np
import pytest
import torch

from oracle import mesh_eval_oracle as O
from simplerecon_b200 import mesh_eval as ME
from tests import mesh_eval_cases as cases
from tests.test_emu_mesh_eval import distances_and_stats, emulated  # noqa: F401  (the fixture)

COLLIDING_N = 32768                  # the smallest power of two with K - w - kMaxProbe well above 0 (157)


def test_colliding_level0_cells_are_kept(emulated):
    """K >= w + kMaxProbe cells homed in one w-slot window force an insert past kMaxProbe slots at level 0.  Level 0
    must still hold every target (its table can take every cell) and settle the queries near them: with a capped
    probe the failed cells' points were dropped from the cell-ordered copy every later level and the brute force
    read, and their distances came out wrong."""
    t, centres, K, w = cases.colliding_level0_set(COLLIDING_N)
    lo, h, n = cases.level0_grid(t)
    cells = np.unique(cases.point_cells(centres, lo, h, n), axis=0)
    H = cases.hash_slots(len(t))
    home = cases.block_hash(cases.block_key(*cells.T), H - 1)
    span = ((home[None, :] - home[:, None]) % H).max(1).min() + 1     # the shortest cyclic window holding them
    assert len(cells) == K and span <= w and K >= w + cases.MAX_PROBE, (len(cells), K, span, w)
    q = cases.queries_near(centres, h, 2000, seed=1)
    d, st = distances_and_stats(q, t)
    np.testing.assert_allclose(d, O.nearest_distances(q, t), rtol=1e-12, atol=0)
    assert st[0] > 0 and st[4] < len(q) // 10, st    # level 0 searched and settled nearly every query


@pytest.mark.parametrize("verts, faces", [pytest.param(v, f, id=name) for name, v, f in cases.sampler_meshes()])
def test_sampler_across_scan_tiles(emulated, verts, faces):
    """Face counts at and past the scan's 2048-element tile, areas over 12 orders of magnitude with zero-area faces
    between them, in face order and shuffled.  A wrong tile carry would pick the wrong triangles while every sample
    still lay on the mesh: the per-face counts of the stratified draw catch it without reproducing the hash, the
    oracle comparison catches it sample by sample."""
    N, seed = 20000, 3
    got = ME.sample_surface(torch.from_numpy(verts), torch.from_numpy(faces), N, seed=seed).numpy()
    areas = cases.triangle_areas(verts, faces)
    assert areas.max() / areas[areas > 0].min() > 1e12 and (areas == 0).any()
    cases.check_stratified_counts(cases.strip_faces_of(got, verts, faces), areas, N)
    face, moved = cases.check_against_oracle(got, verts, faces, N, seed, O)
    assert moved <= 2
    np.testing.assert_array_equal(face, cases.strip_faces_of(got, verts, faces))
