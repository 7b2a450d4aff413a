"""Shared by the mesh-evaluation edge tests (CPU emulation and GPU): seeded numpy constructions of the inputs where
the nearest-distance grid and the sampler of csrc/srcv_mesh_eval.cuh (DESIGN §4.17) take their rare paths — a
level-0 hash table forced past any probe cap, targets that fill a volume, degenerate bounding boxes, and meshes
whose area prefix sum spans several scan tiles."""
from __future__ import annotations

import numpy as np

KEY_BIAS = 1 << 20                  # srcv_block_hash.cuh kKeyBias
MAX_PROBE = 256                     # srcv_mesh_eval.cuh kMaxProbe
SCAN_TILE = 2048                    # srcv_mesh_eval.cuh kTile


def hash_slots(n: int) -> int:
    """The slots of a level's table for n points: the next power of two >= 2 n, at least 1024."""
    h = 1024
    while h < 2 * n:
        h <<= 1
    return h


def block_key(x, y, z) -> np.ndarray:
    u = lambda c: (np.asarray(c, np.int64) + KEY_BIAS).astype(np.uint64)
    return (u(x) << np.uint64(42)) | (u(y) << np.uint64(21)) | u(z)


def block_hash(key: np.ndarray, mask: int) -> np.ndarray:
    k = np.asarray(key, np.uint64).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(31)
        k *= np.uint64(0x7FB5D329728EA185)
        k ^= k >> np.uint64(27)
        k *= np.uint64(0x81DADEF4BC2DD44D)
        k ^= k >> np.uint64(33)
    return (k & np.uint64(mask)).astype(np.int64)


def level0_grid(points: np.ndarray) -> tuple:
    """(lo, h, cells per axis) of level 0 as grid_params_kernel derives them from the fp32 targets, in fp64."""
    p = np.asarray(points, np.float32).astype(np.float64)
    lo, hi = p.min(0), p.max(0)
    e = hi - lo
    S = 2.0 * (e[0] * e[1] + e[1] * e[2] + e[2] * e[0])
    h = np.sqrt(S / len(p)) if S > 0 else e.sum() / len(p)
    h = max(h, e.max() / (KEY_BIAS - 2))
    if not h > 0:
        h = 1.0
    n = np.minimum(np.floor(e * (1.0 / h)).astype(np.int64) + 1, KEY_BIAS - 1)
    return lo, h, n


def point_cells(points: np.ndarray, lo, h, n) -> np.ndarray:
    rel = np.asarray(points, np.float32).astype(np.float64) - lo
    return np.clip(np.floor(rel * (1.0 / h)).astype(np.int64), 0, n - 1)


def colliding_level0_set(n: int, window: int = 64) -> tuple:
    """n targets in the unit cube whose level-0 cells crowd one ``window``-slot stretch of the level-0 table.

    The 8 corners of the cube pin the bounding box, so h = sqrt(6 / n) and the table has hash_slots(n) slots.
    Of all the grid's cells, those whose home slot lies in the fullest window of ``window`` consecutive slots get a
    point at their centre (never on a cell face); the remaining points repeat those centres.  K such cells homed in
    w slots occupy at least K slots from the window's start on, so once K >= w + kMaxProbe some insert must probe
    past kMaxProbe slots, whatever the order of the inserts.  Returns (points (n, 3) fp32, centres (K, 3) fp32,
    K, w)."""
    corners = np.array([[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)], np.float32)
    h = np.sqrt(6.0 / n)
    cells = int(np.floor(1.0 / h)) + 1
    H = hash_slots(n)
    c = np.arange(cells)
    x, y, z = (a.reshape(-1) for a in np.meshgrid(c, c, c, indexing="ij"))
    home = block_hash(block_key(x, y, z), H - 1)
    per_slot = np.bincount(home, minlength=H)
    ring = np.concatenate([per_slot, per_slot[:window]]).cumsum()
    fill = ring[window:] - ring[:-window]                     # homes in slots [s + 1, s + window] (cyclically)
    start = (int(np.argmax(fill)) + 1) % H
    inside = ((home - start) % H) < window
    centres = ((np.stack([x[inside], y[inside], z[inside]], 1) + 0.5) * h).astype(np.float32)
    centres = centres[np.all(centres < 1.0, 1)]               # a last, partial cell may reach past the cube
    K = len(centres)
    if K + 8 > n:
        raise ValueError(f"{K} colliding cells do not fit {n} points")
    rng = np.random.default_rng(n)
    pts = np.concatenate([corners, centres, centres[rng.integers(0, K, n - K - 8)]])
    return pts[rng.permutation(n)], centres, K, window


def queries_near(centres: np.ndarray, h: float, count: int, seed: int) -> np.ndarray:
    """``count`` queries on the given points and within 1.5 h of them."""
    rng = np.random.default_rng(seed)
    q = centres[rng.integers(0, len(centres), count)].astype(np.float64)
    q[count // 4:] += rng.uniform(-1.5 * h, 1.5 * h, size=(count - count // 4, 3))
    return q.astype(np.float32)


def volume_cloud(n: int, num_queries: int, seed: int = 0, outside: float = 0.25) -> tuple:
    """n targets uniform in the unit cube (a predicted cloud full of noise: a coarse level's cells are all occupied,
    not 64^l times fewer as on a surface).  A share ``outside`` of the queries lie 0.02 .. 0.15 outside a face of
    the cube, farther than level 0's kMaxShell + 1 cells once n >= 2^16, so level 0 leaves them open; the rest lie
    inside.  Returns (targets, queries, number of queries outside) — the outside ones come first."""
    rng = np.random.default_rng(seed)
    t = rng.random((n, 3), dtype=np.float32)
    n_out = int(num_queries * outside)
    q = rng.random((num_queries, 3))
    axis = rng.integers(0, 3, n_out)
    gap = rng.uniform(0.02, 0.15, n_out)
    q[np.arange(n_out), axis] = np.where(rng.integers(0, 2, n_out) == 1, 1.0 + gap, -gap)
    return t, q.astype(np.float32), n_out


def collinear(n: int, seed: int = 0) -> np.ndarray:
    """n targets on the x axis between 0 and 10 (two sides of the box are 0: S = 0, h = 10 / n)."""
    rng = np.random.default_rng(seed)
    t = np.zeros((n, 3), np.float32)
    t[:, 0] = rng.uniform(0.0, 10.0, n)
    t[:2, 0] = (0.0, 10.0)
    t[:, 1:] = (1.0, -2.0)
    return t


def coplanar(n: int, seed: int = 0) -> np.ndarray:
    """n targets in the plane z = 0.5 over [0, 4] x [0, 3] (one side of the box is 0)."""
    rng = np.random.default_rng(seed)
    t = np.full((n, 3), 0.5, np.float32)
    t[:, 0] = rng.uniform(0.0, 4.0, n)
    t[:, 1] = rng.uniform(0.0, 3.0, n)
    return t


def far_clusters(n: int, seed: int = 0, apart: float = 1000.0) -> np.ndarray:
    """Two clusters of n / 2 targets, ``apart`` metres apart along x, each 1 mm long in x and w thin in y and z,
    with w = apart n 2^-44 (at most 1 mm): the surface spacing sqrt(2 (ab + bc + ca) / n) ~ sqrt(4 apart w / n) is
    then half of apart / 2^20, so h is widened to the cap of 2^20 - 1 cells per axis and each cluster fills one
    or two cells of level 0."""
    rng = np.random.default_rng(seed)
    w = min(1e-3, apart * n * 2.0 ** -44)
    t = rng.uniform(0.0, 1.0, (n, 3)) * [1e-3, w, w]
    t[n // 2:, 0] += apart
    return t.astype(np.float32)


def all_equal(n: int) -> np.ndarray:
    """n copies of one point (an empty box: h = 1)."""
    return np.tile(np.array([[0.75, -1.25, 2.5]], np.float32), (n, 1))


def lattice(side: int) -> tuple:
    """The integer lattice [0, side)^2 at z = 0 with duplicates up to 2 (side - 1)^2 targets, so that level 0's
    cell edge is exactly sqrt(2 (side - 1)^2 / N) = 1 and every target lies on cell faces; the queries are the
    cell corners of [-2, side + 1]^2 x {-1, 0, 1}.  Returns (targets, queries)."""
    a = np.arange(side, dtype=np.float32)
    lat = np.stack([*np.meshgrid(a, a, indexing="ij"), np.zeros((side, side), np.float32)], -1).reshape(-1, 3)
    n = 2 * (side - 1) ** 2
    t = np.concatenate([lat, lat[np.random.default_rng(side).integers(0, len(lat), n - len(lat))]])
    b = np.arange(-2, side + 2, dtype=np.float32)
    q = np.stack(np.meshgrid(b, b, np.array([-1.0, 0.0, 1.0], np.float32), indexing="ij"), -1).reshape(-1, 3)
    return t, q


# ---- the sampler ----------------------------------------------------------------------------------------

def strip_mesh(num_faces: int, seed: int, shuffle: bool = False, zero_every: int = 7) -> tuple:
    """``num_faces`` disjoint right triangles on a square grid of the x-z plane within [0, 4) m, each with one leg
    of d / 2 along x (d the grid spacing) and one of 10^-13 .. 1 m (log-uniform, both ends present) along y from
    y = 0, where fp32 keeps it to full relative precision: areas span 13 orders of magnitude.  Every
    ``zero_every``-th triangle is degenerate (its third vertex on the x leg: zero area).  Faces in grid order, or
    shuffled.  Returns (verts (3F, 3) fp32, faces (F, 3) int32)."""
    rng = np.random.default_rng(seed)
    F = num_faces
    G = int(np.ceil(np.sqrt(F)))
    d = 4.0 / G
    k = np.arange(F)
    a = np.stack([(k % G) * d, np.zeros(F), (k // G) * d], 1)
    b = a + [d / 2, 0.0, 0.0]
    leg = 10.0 ** rng.uniform(-13.0, 0.0, F)
    leg[1:3] = (1.0, 1e-13)
    c = a + np.stack([np.zeros(F), leg, np.zeros(F)], 1)
    c[::zero_every] = (a[::zero_every] + b[::zero_every]) * 0.5
    verts = np.stack([a, b, c], 1).reshape(-1, 3).astype(np.float32)
    faces = np.arange(3 * F, dtype=np.int32).reshape(F, 3)
    if shuffle:
        faces = faces[rng.permutation(F)]
    return verts, faces


def strip_faces_of(samples: np.ndarray, verts: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """The face of a strip mesh each sample lies in, from its position alone (the triangles sit in disjoint cells
    of the grid; within its cell a triangle covers x in [0, d / 2] and y >= 0); -1 where it lies in none."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    F = len(f)
    G = int(np.ceil(np.sqrt(F)))
    d = 4.0 / G
    s = np.asarray(samples, np.float64)
    ix, iz = np.floor(s[:, 0] / d + 0.25).astype(np.int64), np.rint(s[:, 2] / d).astype(np.int64)
    cell = np.where((ix >= 0) & (ix < G) & (iz >= 0), iz * G + ix, -1)
    of_cell = np.full(G * G, -1, np.int64)
    of_cell[f[:, 0] // 3] = np.arange(F)                     # vertex 3k is the corner of grid cell k
    face = np.where((cell >= 0) & (cell < G * G), of_cell[np.clip(cell, 0, G * G - 1)], -1)
    ok = face >= 0
    a = v[f[np.maximum(face, 0), 0]]
    ok &= (s[:, 1] >= 0) & (s[:, 0] >= a[:, 0] - 1e-6) & (s[:, 0] <= a[:, 0] + d / 2 + 1e-6) & \
          (np.abs(s[:, 2] - a[:, 2]) <= 1e-6)
    return np.where(ok, face, -1)


# face counts around the scan's tile of 2048, the last a few elements into a fourth tile, in face order and shuffled;
# the large one (GPU only) about 10^6 faces, shuffled
SAMPLER_MESHES = ("strip2047", "strip2048", "strip2049", f"strip{3 * SCAN_TILE + 5}",
                  f"strip{3 * SCAN_TILE + 5}_shuffled")
LARGE_SAMPLER_MESH = "strip1000003_shuffled"


def sampler_mesh(name: str) -> tuple:
    """The strip mesh called ``name`` ("strip<F>" or "strip<F>_shuffled"), seeded by F."""
    F = int(name.removeprefix("strip").removesuffix("_shuffled"))
    return strip_mesh(F, seed=F, shuffle=name.endswith("_shuffled"))


def sampler_meshes(large: bool = False) -> list:
    """[(name, verts, faces)] of SAMPLER_MESHES, and with ``large`` LARGE_SAMPLER_MESH (the GPU tests add the fused
    room mesh, which needs the device to build)."""
    return [(n, *sampler_mesh(n)) for n in SAMPLER_MESHES + ((LARGE_SAMPLER_MESH,) if large else ())]


def triangle_areas(verts: np.ndarray, faces: np.ndarray) -> np.ndarray:
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)


def check_stratified_counts(face: np.ndarray, areas: np.ndarray, N: int) -> None:
    """Each face holds within 2 of N A_f / A samples (sample i is drawn from the i-th N-th of the area), a face
    of zero area none, and the counts add up to N."""
    assert face.min() >= 0
    counts = np.bincount(face, minlength=len(areas))
    assert counts.sum() == N
    expect = N * areas / areas.sum()
    bad = np.flatnonzero(np.abs(counts - expect) > 2.0)
    assert len(bad) == 0, (bad[:5], counts[bad[:5]], expect[bad[:5]])
    assert not counts[areas == 0.0].any()


def check_against_oracle(got: np.ndarray, verts: np.ndarray, faces: np.ndarray, N: int, seed: int, oracle) -> tuple:
    """The kernel's samples against ``oracle.sample_surface(..., return_faces=True)``: equal within 1e-6 m, except
    where the draw t_i lies within F 2^-52 total of a boundary of the oracle's CDF (the kernel's tiled prefix sum
    and the sequential cumsum may round a boundary differently and so pick the triangle on its other side); such
    a sample must be the oracle's point on that neighbouring triangle (the next one of non-zero area) with the
    same barycentric weights.  Returns (the kernel's face of every sample, the number of neighbour picks)."""
    ref, tri = oracle.sample_surface(verts, faces, N, seed=seed, return_faces=True)
    face = tri.copy()
    bad = np.flatnonzero(np.abs(got.astype(np.float64) - ref).max(1) > 1e-6)
    if len(bad) == 0:
        return face, 0
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    areas = triangle_areas(verts, faces)
    cdf = np.cumsum(areas)
    total = cdf[-1]
    i = bad.astype(np.uint64)
    t = (i.astype(np.float64) + oracle.uniforms(seed, i, 0)) / float(N) * total
    t = np.where(t < total, t, total * (1.0 - 2.0 ** -52))
    tol = len(f) * 2.0 ** -52 * total
    k = tri[bad]
    nz = np.flatnonzero(areas > 0)
    pos = np.searchsorted(nz, k)
    below, above = nz[np.maximum(pos - 1, 0)], nz[np.minimum(pos + 1, len(nz) - 1)]
    s = np.sqrt(oracle.uniforms(seed, i, 1))
    u2 = oracle.uniforms(seed, i, 2)
    w = np.stack([1.0 - s, s * (1.0 - u2), s * u2], 1)

    def point_on(tr):
        return np.einsum("nk,nkd->nd", w, v[f[tr]]).astype(np.float32).astype(np.float64)

    near_lo = (pos > 0) & (np.abs(t - cdf[below]) <= tol)      # the boundary below the oracle's triangle
    near_hi = (pos < len(nz) - 1) & (np.abs(t - cdf[k]) <= tol)  # the boundary above it
    g = got[bad].astype(np.float64)
    on_lo = near_lo & (np.abs(g - point_on(below)).max(1) <= 1e-6)
    on_hi = near_hi & (np.abs(g - point_on(above)).max(1) <= 1e-6)
    ok = on_lo | on_hi
    assert np.all(ok), (bad[~ok][:5], t[~ok][:5], k[~ok][:5])
    face[bad] = np.where(on_lo, below, above)
    return face, len(bad)
