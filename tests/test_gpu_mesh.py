"""GPU: the marching-cubes mesh extraction kernel (csrc/srcv_mesh.cuh) through TSDF.extract_mesh, against
the fp64 oracle at larger sizes, deterministic, and at OurFuser's default full size (±10 m at 4 cm)."""
import numpy as np
import pytest
import torch

import simplerecon_b200 as S
from oracle import mesh_oracle as M
from simplerecon_b200 import _native
from simplerecon_b200.synthetic import make_tsdf_case
from tests.test_emu_mesh import every_face_in_a_weighted_cube

pytestmark = pytest.mark.gpu


def check_against_oracle(vol, scale_to_world, single_mesh):
    verts, faces, normals = vol.extract_mesh(scale_to_world=scale_to_world, single_mesh=single_mesh)
    assert verts.device.type == "cuda" and faces.device.type == "cuda" and normals.device.type == "cuda"
    origin_h = vol.origin.half().double().numpy()
    ov, of, on = M.extract(vol.tsdf_values.cpu(), vol.tsdf_weights.cpu(), scale_to_world=scale_to_world,
                           single_mesh=single_mesh, origin=origin_h, voxel_size=vol.voxel_size)
    assert verts.shape == ov.shape and faces.shape == of.shape
    assert np.array_equal(faces.cpu().numpy().astype(np.int64), of)
    kv = verts.cpu().numpy().astype(np.float64)
    mag = np.abs(ov)
    if scale_to_world:
        mag = np.maximum(np.maximum(mag, np.abs(origin_h)[None]), np.abs(ov - origin_h[None]))
    assert (np.abs(kv - ov) <= 4 * np.spacing(mag.astype(np.float32)).astype(np.float64)).all()
    assert np.abs(normals.cpu().numpy() - on).max(initial=0.0) <= 1e-5
    return verts, faces, normals


def _sphere(dims):
    x, y, z = np.meshgrid(*[np.arange(k, dtype=np.float64) for k in dims], indexing="ij")
    c = [d / 2 - 0.41 for d in dims]
    f = (np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - (min(dims) / 2 - 4.3)) / 3.0
    f += 0.3 * np.sin(x / 2.3) * np.cos(y / 3.1)
    values = torch.from_numpy(np.clip(f, -1, 1)).half().cuda()
    weights = torch.from_numpy(np.abs(f) < 1.5).half().cuda()
    return S.TSDF(values, weights, 0.04, torch.tensor([-2.37, 1.11, 0.52]))


def _fused_room(seed, voxel, frames=4, hw=(96, 128)):
    c = make_tsdf_case(seed=seed, frames=frames, voxel_size=voxel, height=hw[0], width=hw[1])
    vol = S.TSDF.from_bounds(c["bounds"], voxel)
    S.TSDFFuser(vol, max_depth=c["max_depth"]).integrate_depth(c["depth"].cuda(), c["cam_T_world"].cuda(), c["K"].cuda())
    return vol


@pytest.mark.parametrize("scale_to_world,single_mesh", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("case", ["sphere_vec", "sphere_scalar", "room"])
def test_matches_oracle(cuda_device, case, scale_to_world, single_mesh):
    vol = {"sphere_vec": lambda: _sphere((72, 64, 80)), "sphere_scalar": lambda: _sphere((61, 50, 45)),
           "room": lambda: _fused_room(41, 0.04)}[case]()
    _, faces, _ = check_against_oracle(vol, scale_to_world, single_mesh)
    assert len(faces) > 5000


def test_deterministic_variant_and_launches(cuda_device):
    vol = _fused_room(42, 0.05)
    n0 = _native.launch_count()
    a = vol.extract_mesh(single_mesh=True)
    assert _native.launch_count() - n0 == 4 and _native.last_variant() == "tsdf_mesh_mc"
    b = vol.extract_mesh(single_mesh=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_full_size_volume(cuda_device):
    """OurFuser's default volume (±10 m at 4 cm: 504^3) with the synthetic room fused from 8 frames."""
    c = make_tsdf_case(seed=21, frames=8, voxel_size=0.04, height=240, width=320, room=(6.0, 5.0, 3.0))
    bounds = {k: (-10.0 if k.endswith("min") else 10.0) for k in ("xmin", "xmax", "ymin", "ymax", "zmin", "zmax")}
    vol = S.TSDF.from_bounds(bounds, 0.04)
    assert tuple(vol.tsdf_values.shape) == (504, 504, 504)
    S.TSDFFuser(vol, max_depth=3.0).integrate_depth(c["depth"].cuda(), c["cam_T_world"].cuda(), c["K"].cuda())
    verts, faces, normals = vol.extract_mesh()
    assert len(verts) == M.crossing_edges_torch(vol.tsdf_values)
    assert len(faces) > 100000 and torch.isfinite(verts).all() and torch.isfinite(normals).all()
    # closed and consistently oriented (the fused region does not reach the volume border).  Exact
    # zeros put several edge vertices on one grid point and drop the degenerate faces there, so edges
    # with an endpoint on a grid point are left out of the count.
    vi, fi, _ = vol.extract_mesh(scale_to_world=False)
    assert torch.equal(fi, faces)
    on_grid = (vi == vi.round()).all(1)
    f = faces.long()
    d = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    d = d[~(on_grid[d[:, 0]] | on_grid[d[:, 1]])]
    assert len(d) > 0.9 * 3 * len(f)
    key = d[:, 0] * len(verts) + d[:, 1]
    assert len(torch.unique(key)) == len(key)                          # every directed edge once
    und = torch.sort(d, 1).values
    _, cnt = torch.unique(und[:, 0] * len(verts) + und[:, 1], return_counts=True)
    assert bool((cnt == 2).all())                                      # every undirected edge twice
    v1, f1, _ = vol.extract_mesh(scale_to_world=False, single_mesh=True)
    assert 0 < len(f1) < len(faces)
    assert every_face_in_a_weighted_cube(vol.tsdf_weights, v1.cpu().numpy(), f1.cpu().numpy())
