"""CPU: the mesh-export surface of the TSDF mirror against the unmodified reference (tools/tsdf.py),
from stored outputs (tests/refgolden.py, written by tests/golden/make_mesh_reference_golden.py):
  - TSDF.from_mesh gives the reference's dims and origin;
  - the reference's to_mesh(scale_to_world=True), run with skimage's marching_cubes replaced by the
    oracle (oracle/mesh_oracle.py) and trimesh.Trimesh by a recorder, gives the world vertices and
    faces that extract_mesh(scale_to_world=True) produces: this pins the fp16-origin arithmetic."""
import types

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as M
from simplerecon_b200 import tsdf as tsdf_mod
from tests import refgolden
from tests.test_emu_mesh import emulated  # noqa: F401  (fixture)

MESH_CASES = [(0, 0.04, (-1.37, 2.21, -0.73)), (1, 0.05, (3.3, -9.99, 0.31))]
BOUNDS_CASES = [(0, 0.04), (1, 0.1), (2, 0.013)]


def _volume(seed):
    g = np.random.default_rng(seed)
    n = (19, 17, 24)
    x, y, z = np.meshgrid(*[np.arange(k, dtype=np.float64) for k in n], indexing="ij")
    c = np.array(n) / 2 + g.uniform(-1, 1, 3)
    f = (np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - 6.3) / 3.0
    return torch.from_numpy(np.clip(f, -1, 1)).half()


def _mesh_vertices(seed):
    g = np.random.default_rng(100 + seed)
    return g.uniform(-3, 4, (50, 3)) * np.array([1.0, 0.7, 0.4])


def reference_outputs():
    """For tests/golden/make_mesh_reference_golden.py."""
    from oracle.ref_import import load_reference_tsdf
    R = load_reference_tsdf()
    out = {}
    for seed, voxel in BOUNDS_CASES:
        ref = R.TSDF.from_mesh(types.SimpleNamespace(vertices=_mesh_vertices(seed)), voxel_size=voxel)
        out[f"bounds_{seed}"] = {"dims": torch.tensor(ref.tsdf_values.shape), "origin": ref.origin.clone()}
    calls = []
    R.module.trimesh = types.SimpleNamespace(Trimesh=lambda vertices, faces, normals: calls.append((vertices, faces)))
    R.module.measure = types.SimpleNamespace(
        marching_cubes=lambda v, level, allow_degenerate: (lambda o: (o[0].astype(np.float32), o[1], o[2], None))(
            M.extract(torch.from_numpy(v).half())))
    for seed, voxel, origin in MESH_CASES:
        vals = _volume(seed)
        o = torch.tensor(origin, dtype=torch.float32)
        ref = R.TSDF(R.TSDF.generate_voxel_coords(o, tuple(vals.shape), voxel), vals, torch.ones_like(vals), voxel, o)
        calls.clear()
        ref.to_mesh(scale_to_world=True)
        verts, faces = calls[0]
        out[f"mesh_{seed}"] = {"verts": torch.as_tensor(verts).float(), "faces": torch.as_tensor(faces)}
    return out


@pytest.mark.parametrize("seed,voxel", BOUNDS_CASES)
def test_from_mesh_matches_reference(seed, voxel):
    G = refgolden.load("mesh_vs_reference", f"bounds_{seed}")
    ours = tsdf_mod.TSDF.from_mesh(types.SimpleNamespace(vertices=_mesh_vertices(seed)), voxel, device="cpu")
    assert tuple(ours.tsdf_values.shape) == tuple(G["dims"].tolist())
    assert torch.equal(ours.origin.half(), G["origin"])      # the reference keeps the origin in fp16


@pytest.mark.parametrize("seed,voxel,origin", MESH_CASES)
def test_to_mesh_world_vertices_match_reference(emulated, seed, voxel, origin):  # noqa: F811
    G = refgolden.load("mesh_vs_reference", f"mesh_{seed}")
    vals = _volume(seed)
    vol = tsdf_mod.TSDF(vals, torch.ones_like(vals), voxel, torch.tensor(origin, dtype=torch.float32))
    verts, faces, _ = vol.extract_mesh(scale_to_world=True)
    assert torch.equal(faces.long(), G["faces"].long())
    # the reference's world arithmetic on the index-space vertices: half origin + fp32 v * voxel_size
    vi, _, _ = vol.extract_mesh(scale_to_world=False)
    ref_world = G["verts"]
    oh = torch.tensor(origin).half().float()
    assert torch.equal(verts, oh[None] + vi * voxel)
    mag = torch.maximum(ref_world.abs(), oh.abs()[None].expand_as(ref_world)).numpy()
    tol = torch.from_numpy(4 * np.spacing(np.maximum(mag, np.abs(vi.numpy() * voxel))).astype(np.float32))
    assert ((verts - ref_world).abs() <= tol).all()
