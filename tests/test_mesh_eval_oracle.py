"""CPU: the numpy / scipy oracle of the mesh evaluation (oracle/mesh_eval_oracle.py, DESIGN §4.17) — KD-tree
distances against brute force, hand cases of the six metrics, and the sampler's area distribution."""
import numpy as np
import pytest
from scipy import stats

from oracle import mesh_eval_oracle as O


def test_kdtree_matches_brute_force():
    rng = np.random.default_rng(0)
    for n, m in ((1, 7), (50, 300), (400, 257)):
        p = rng.normal(size=(n, 3)).astype(np.float32)
        q = (rng.normal(size=(m, 3)) * 2).astype(np.float32)
        np.testing.assert_array_equal(O.nearest_distances(q, p), O.brute_distances(q, p))


def _grid(z: float, n: int = 20, spacing: float = 0.1) -> np.ndarray:
    x, y = np.meshgrid(np.arange(n) * spacing, np.arange(n) * spacing, indexing="ij")
    return np.stack([x.ravel(), y.ravel(), np.full(n * n, z)], 1).astype(np.float32)


@pytest.mark.parametrize("offset,share", [(0.03, 1.0), (0.07, 0.0)])
def test_offset_grids(offset, share):
    """Two identical grids (10 cm spacing) offset along their normal: every distance is the offset evaluated in
    fp64 from the fp32 coordinates; at 3 cm both shares are 1, at 7 cm both are 0 and the F-score is 0."""
    a, b = _grid(1.0), _grid(1.0 + offset)
    d = np.float64(np.float32(1.0 + offset)) - np.float64(np.float32(1.0))
    np.testing.assert_array_equal(O.nearest_distances(a, b), np.full(len(a), d))
    np.testing.assert_array_equal(O.nearest_distances(b, a), np.full(len(a), d))
    m = O.mesh_metrics(a, b, threshold=0.05)
    assert list(m) == list(O.KEYS)
    assert m["acc"] == m["comp"] == m["chamfer"] == d
    assert m["precision"] == m["recall"] == m["fscore"] == share


def test_fscore_of_unequal_shares():
    d_pred, d_gt = np.array([0.01, 0.02, 0.2, 0.3]), np.array([0.01, 0.5])
    m = O.metrics_from_distances(d_pred, d_gt, 0.05)
    assert (m["precision"], m["recall"]) == (0.5, 0.5) and m["fscore"] == 0.5
    assert m["acc"] == pytest.approx(0.1325) and m["comp"] == pytest.approx(0.255)


def test_uniforms_are_uniform_and_seeded():
    i = np.arange(200000)
    u = O.uniforms(0, i, 0)
    assert 0.0 <= u.min() and u.max() < 1.0
    assert stats.kstest(u, "uniform").pvalue > 1e-3
    assert not np.array_equal(u, O.uniforms(1, i, 0)) and not np.array_equal(u, O.uniforms(0, i, 1))
    np.testing.assert_array_equal(u, O.uniforms(0, i, 0))


def test_sampler_area_distribution_chi_square():
    """A mesh of very unequal triangles: the share of samples per triangle follows the areas."""
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [10, 0, 0], [10, 1e-3, 0], [10, 0, 1e-3],
                      [0, 0, 5], [3, 0, 5], [0, 4, 5]], np.float32)
    faces = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8], [0, 1, 6]], np.int64)
    n = 100000
    pts, tri = O.sample_surface(verts, faces, n, seed=3, return_faces=True)
    area = O.triangle_areas(verts, faces)
    expected = n * area / area.sum()
    observed = np.bincount(tri, minlength=len(faces))
    assert stats.chisquare(observed, expected).pvalue > 1e-3
    # every sample lies on its triangle: barycentric weights in [0, 1] reproduce it
    v = verts.astype(np.float64)
    a, b, c = v[faces[tri, 0]], v[faces[tri, 1]], v[faces[tri, 2]]
    nrm = np.cross(b - a, c - a)
    off = np.abs(((pts - a) * nrm).sum(1)) / np.linalg.norm(nrm, axis=1)
    assert off.max() < 1e-5
    # stratified: triangle order follows sample order
    assert np.all(np.diff(tri) >= 0)
