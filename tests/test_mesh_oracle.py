"""CPU: the generated marching-cubes table and the mesh oracle's geometry (DESIGN §4.10).

The table is regenerated and compared with the committed header; the oracle (oracle/mesh_oracle.py,
the restatement the kernel is tested against) is checked on analytic fields for closedness,
orientation, topology and accuracy, and on a field with many exact zeros."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as M

ROOT = Path(__file__).resolve().parents[1]


def _gen():
    spec = importlib.util.spec_from_file_location("gen_mc_table", ROOT / "scripts" / "gen_mc_table.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---- the table ---------------------------------------------------------------------------------

def test_table_header_is_regenerated_identically():
    assert _gen().render() == (ROOT / "simplerecon_b200" / "csrc" / "srcv_mc_table.h").read_text()


def test_table_uses_exactly_the_crossing_edges():
    g = _gen()
    tab = M.read_table()
    for case in range(256):
        crossing = {e for e in range(12) if ((case >> g.edge_corners(e)[0]) & 1) != ((case >> g.edge_corners(e)[1]) & 1)}
        used = {int(e) for e in tab[case].reshape(-1) if e >= 0}
        assert used == crossing, case
        assert [tuple(t) for t in tab[case] if t[0] >= 0] == g.triangles(case)


def test_loop_edges_lie_on_cube_faces():
    g = _gen()
    for case in range(256):
        for loop in g.loops(case):
            for a, b in zip(loop, loop[1:] + loop[:1]):
                assert any(a in f and b in f for f in g.FACE_EDGES), (case, loop)


# ---- mesh checks -------------------------------------------------------------------------------

def _volume(field: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.clip(field, -1, 1)).half()


def _grid(n):
    return np.meshgrid(*[np.arange(k, dtype=np.float64) for k in n], indexing="ij")


def mesh_stats(verts, faces):
    """closed (every undirected edge in two faces, every directed edge once), chi, components."""
    f = np.asarray(faces)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    directed_unique = len(np.unique(d, axis=0)) == len(d)
    und, cnt = np.unique(np.sort(d, 1), axis=0, return_counts=True)
    closed = bool((cnt == 2).all()) and directed_unique
    used = np.unique(f)
    chi = len(used) - len(und) + len(f)
    # components by union-find over the used vertices
    parent = {int(v): int(v) for v in used}

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a
    for a, b in und:
        ra, rb = find(int(a)), find(int(b))
        if ra != rb:
            parent[ra] = rb
    comps = len({find(int(v)) for v in used})
    return closed, chi, comps


def enclosed_volume_area(verts, faces):
    p = np.asarray(verts)[np.asarray(faces)]
    vol = np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0
    area = 0.5 * np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1).sum()
    return vol, area


def sphere_field(n, c, r):
    x, y, z = _grid(n)
    return (np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - r) / 4.0


def _no_exact_zero(vol):
    assert not bool((vol == 0).any())
    return vol


def test_sphere_closed_genus0_accurate():
    r, c = 12.3, (20.4, 19.7, 21.1)
    vol = _no_exact_zero(_volume(sphere_field((42, 41, 43), c, r)))
    verts, faces, normals = M.extract(vol)
    closed, chi, comps = mesh_stats(verts, faces)
    assert closed and chi == 2 and comps == 1
    v, a = enclosed_volume_area(verts, faces)
    assert v > 0                                        # outward (toward increasing values) winding
    assert abs(v / (4 / 3 * np.pi * r ** 3) - 1) < 0.01
    assert abs(a / (4 * np.pi * r ** 2) - 1) < 0.02
    dist = np.linalg.norm(verts - np.array(c), axis=1) - r
    assert np.abs(dist).max() < 0.05
    # face normals (winding) agree with the interpolated vertex normals
    p = verts[faces]
    fn = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    big = np.linalg.norm(fn, axis=1) > 1e-3
    agree = np.einsum("ij,ij->i", fn[big], normals[faces[big]].sum(1)) > 0
    assert agree.mean() >= 0.99


def test_torus_has_euler_characteristic_zero():
    x, y, z = _grid((44, 44, 24))
    R, r = 12.2, 4.6
    q = np.sqrt((x - 21.7) ** 2 + (y - 22.1) ** 2) - R
    vol = _no_exact_zero(_volume((np.sqrt(q ** 2 + (z - 11.6) ** 2) - r) / 3.0))
    verts, faces, _ = M.extract(vol)
    closed, chi, comps = mesh_stats(verts, faces)
    assert closed and chi == 0 and comps == 1


def test_two_spheres_two_components():
    f = np.minimum(sphere_field((40, 30, 30), (10.3, 14.6, 15.2), 7.1), sphere_field((40, 30, 30), (28.8, 15.4, 14.1), 6.3))
    verts, faces, _ = M.extract(_no_exact_zero(_volume(f)))
    closed, chi, comps = mesh_stats(verts, faces)
    assert closed and comps == 2 and chi == 4


def random_smooth_field(seed, n=(22, 20, 18)):
    """A smooth random field, positive at the border, crossing zero often."""
    g = np.random.default_rng(seed)
    f = g.standard_normal(n)
    for ax in range(3):                              # separable smoothing
        f = (np.roll(f, 1, ax) + 2 * f + np.roll(f, -1, ax)) / 4
    f = f / f.std() * 0.5 + g.uniform(-0.2, 0.2)
    f[0], f[-1], f[:, 0], f[:, -1], f[:, :, 0], f[:, :, -1] = 1, 1, 1, 1, 1, 1
    vol = _volume(f)
    vol[vol == 0] = 0.001                             # no exact zeros
    return vol


@pytest.mark.parametrize("seed", range(24))
def test_random_fields_closed_and_oriented(seed):
    vol = random_smooth_field(seed)
    verts, faces, normals = M.extract(vol)
    assert len(faces) > 50
    closed, _, _ = mesh_stats(verts, faces)
    assert closed
    p = verts[faces]
    fn = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    big = np.linalg.norm(fn, axis=1) > 1e-2
    agree = np.einsum("ij,ij->i", fn[big], normals[faces[big]].sum(1)) > 0
    assert agree.mean() >= 0.95


def test_random_fields_exercise_every_ambiguous_face():
    """Across the random fields, every ambiguous face pattern occurs on every face orientation."""
    seen = set()
    for seed in range(24):
        ins = (random_smooth_field(seed).float() < 0).numpy()
        for a in range(3):
            b, c = [k for k in range(3) if k != a]
            s = np.moveaxis(ins, (a, b, c), (0, 1, 2))
            q00, q10, q01, q11 = s[:, :-1, :-1], s[:, 1:, :-1], s[:, :-1, 1:], s[:, 1:, 1:]
            if ((q00 & q11) & ~(q10 | q01)).any():
                seen.add((a, 0))
            if ((q10 & q01) & ~(q00 | q11)).any():
                seen.add((a, 1))
    assert seen == {(a, d) for a in range(3) for d in range(2)}


def exact_zero_field():
    x, y, z = _grid((30, 28, 26))
    f = np.sin(x / 3.1) + np.cos(y / 2.7) + np.sin(z / 3.7 + 0.4) - 0.2
    return torch.from_numpy(np.round(np.clip(f, -1, 1) * 4) / 4).half()     # quantised: many exact zeros


def test_exact_zeros_no_degenerate_faces_no_nan():
    vol = exact_zero_field()
    assert int((vol == 0).sum()) > 500
    verts, faces, normals = M.extract(vol)
    assert np.isfinite(verts).all() and np.isfinite(normals).all()
    assert len(verts) == M.crossing_edges_torch(vol)
    p = verts[faces].astype(np.float32)
    assert not (np.all(p[:, 0] == p[:, 1], -1) | np.all(p[:, 1] == p[:, 2], -1) | np.all(p[:, 0] == p[:, 2], -1)).any()
    assert len(faces) > 100
