"""GPU: every compile-time instantiation of the two forward sweeps against the oracle.

The launchers pick a template instantiation from the feature-map size, the planes mode and (dot
sweep) the warp-tile width:

* `dot_fast_kernel<PER_PIXEL, TW, TH, kTileW>` (csrc/srcv_dot.cu, `launch_fast_sized`): the sizes of
  the `SRCV_SIZED(W, H)` list plus the run-time-size form `<..., 0, 0, ...>`, per-plane and per-pixel
  planes, warp tiles 16 x 2 and 32 x 1 (`SRCV_DOT_TILE_W`, read once per process).  The launcher also
  splits the plane loop over CTAs when a frame has few warps; a split sweep ends in the last-arriver
  argmax, an unsplit one fuses the argmax.
* `mlp_tc_kernel<PER_PIXEL, TW, TH>` (csrc/srcv_mlp_tc.cu, `SRCV_TC_LAUNCH(PP, W, H)`): the same idea
  for the wgmma metadata-MLP sweep.

With a compile-time size every gather offset is an immediate, so each instantiation has its own address
arithmetic, and a wrong stride in one of them shows only at that map size.  MATRIX below names one row
per (kernel, size, planes mode, tile) and the B, D and H x W that reach it;
tests/test_emu_instantiations.py parses the dispatch lists and fails when an instantiation has no row.

Judged against the oracle's fp64 evaluation (tests/parity.py): from 96 x 128 up the oracle's own fp32
result is further from fp64 than the kernels are, so the fp32 oracle alone would give false failures.
Oracle work stays small (hero: B = 1, D <= 5); full-D runs are checked through exact properties:
per-pixel planes holding the per-plane values give the per-plane result bit for bit, the 32 x 1 warp
tile gives the 16 x 2 tile's result bit for bit (each thread computes its own pixel in the same order
whatever the warp shape), shard invariance and determinism.
"""
from __future__ import annotations

import os
import subprocess
import sys
from dataclasses import dataclass, replace
from pathlib import Path

import pytest
import torch

import simplerecon_b200 as S
from oracle import costvolume_oracle as O
from simplerecon_b200 import _native
from simplerecon_b200.synthetic import make_tuple, mlp_state, to_device
from tests.parity import assert_cost_close, assert_lowest_close, assert_mask_close, cost_tol

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


# --------------------------------------------------------------------------------------------- #
# the instantiation matrix                                                                       #
# --------------------------------------------------------------------------------------------- #
@dataclass(frozen=True)
class Row:
    kernel: str          # "dot": dot_fast_kernel, "hero": mlp_tc_kernel
    inst: tuple          # (TW, TH) template arguments: compile-time map size, (0, 0) = run-time form
    per_pixel: bool      # PER_PIXEL template argument: (B, D, H, W) planes; else per-plane / range planes
    tile: int            # dot: kTileW, the warp-tile width SRCV_DOT_TILE_W selects; hero: 0
    B: int
    D: int
    H: int
    W: int
    split: bool = False  # dot: the launcher splits the plane loop (last-arriver argmax)

    @property
    def id(self) -> str:
        tw, th = self.inst
        size = f"{tw}x{th}" if tw else "rt"
        planes = "pixel" if self.per_pixel else "plane"
        tile = f",tile{self.tile}" if self.kernel == "dot" else ""
        split = ("-split" if self.split else "-fused") if self.kernel == "dot" else ""
        return f"{self.kernel}<{size},{planes}{tile}>-B{self.B}-D{self.D}-{self.H}x{self.W}{split}"


# (template size, H, W): the last one is a ragged map that takes the run-time-size form
DOT_MAPS = [((160, 120), 120, 160), ((128, 96), 96, 128), ((64, 48), 48, 64), ((0, 0), 37, 53)]
HERO_MAPS = [((160, 120), 120, 160), ((128, 96), 96, 128), ((0, 0), 37, 53)]
# dot: D = 8 never splits (D / 2 < 2 * kDC); B = 1 at D = 64 leaves so few warps that it splits 8 ways
DOT_PLANES = [(2, 8, False), (1, 64, True)]

MATRIX = [Row("dot", inst, pp, tile, B, D, H, W, split)
          for inst, H, W in DOT_MAPS for pp in (False, True) for tile in (16, 32) for B, D, split in DOT_PLANES]
# hero: an even D and an odd D (a partial two-plane tile that holds the last, mask-carrying plane)
MATRIX += [Row("hero", inst, pp, 0, 1, D, H, W)
           for inst, H, W in HERO_MAPS for pp in (False, True) for D in ((4, 5) if inst[0] else (2, 3))]

HERO_K, DOT_K, C = 7, 7, 16
DOT_WARPS_PER_SM = 128          # launch_dot_fast's default occupancy target (SRCV_DOT_WARPS_PER_SM)


def dot_plane_split(B, D, H, W, tile, sms, want=DOT_WARPS_PER_SM):
    """launch_dot_fast's plane-loop split, restated: the number of CTAs a plane column is cut into."""
    tile_h, warps_per_cta, kdc = 32 // tile, 2, 4
    warps = B * -(-W // tile) * -(-H // (tile_h * warps_per_cta)) * warps_per_cta
    s = 1
    while s < 8 and warps * s < want * sms and D // (s * 2) >= 2 * kdc:
        s *= 2
    return s


def _seed(row):
    return 1009 * row.H + 31 * row.W + 7 * row.D + row.B + (500 if row.per_pixel else 0) + (3 if row.kernel == "hero" else 0)


def row_inputs(row):
    """Seeded inputs of a row (independent of the warp tile, so both tiles see the same call)."""
    K = DOT_K if row.kernel == "dot" else HERO_K
    t = make_tuple(row.B, K, row.H, row.W, channels=C, seed=_seed(row))
    planes = None
    if row.per_pixel:
        g = torch.Generator().manual_seed(_seed(row) + 1)
        planes = 0.3 + 4.0 * torch.rand(row.B, row.D, row.H, row.W, generator=g)
    return t, planes


def _mlp_manager(H, W, D, sd, fast_cls=False):
    cls = S.FastFeatureVolumeManager if fast_cls else S.FeatureVolumeManager
    m = cls(H, W, num_depth_bins=D, mlp_channels=[0, 128, 128, 1], matching_dim_size=C, num_source_views=HERO_K)
    m.load_state_dict({**m.state_dict(), **sd})
    return m.cuda().eval()


def run(kind, t, D, planes=None, sd=None, variant=_native.VARIANT_AUTO, fast_cls=False):
    """One inference call through the manager classes -> ((cost, lowest, planes, mask), variant used)."""
    B, K, _, H, W = t["src_feats"].shape
    m = S.CostVolumeManager(H, W, num_depth_bins=D).cuda().eval() if kind == "dot" else \
        _mlp_manager(H, W, D, sd, fast_cls)
    _native.set_variant(variant)
    try:
        with torch.inference_mode():
            out = m(**to_device(t, "cuda"), depth_planes_bdhw=None if planes is None else planes.cuda(),
                    return_mask=kind != "dot")
        torch.cuda.synchronize()
        return out, _native.last_variant()
    finally:
        _native.set_variant(_native.VARIANT_AUTO)


def process_tile():
    """The warp tile this process's dot sweep uses (launch_dot_fast latches it on its first call).
    The tile is not observable through the API, so the tests rely on the environment variable."""
    return 32 if os.environ.get("SRCV_DOT_TILE_W", "").strip() == "32" else 16


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fp64(t, planes):
    return {k: v.double() for k, v in t.items()}, None if planes is None else planes.double()


def _argmax_is_lowest(cost, planes, lowest):
    idx = cost.argmax(1, keepdim=True)
    assert torch.equal(torch.gather(planes.expand_as(cost), 1, idx).squeeze(1), lowest)


@pytest.fixture(autouse=True)
def _device(cuda_device):
    yield


# --------------------------------------------------------------------------------------------- #
# dot sweep                                                                                      #
# --------------------------------------------------------------------------------------------- #
def run_dot_row(row):
    assert row.tile == process_tile(), f"{row.id}: this process runs warp tile {process_tile()}"
    if "SRCV_DOT_WARPS_PER_SM" not in os.environ:
        assert (dot_plane_split(row.B, row.D, row.H, row.W, row.tile, _sms()) > 1) == row.split, row.id
    t, planes = row_inputs(row)
    out, used = run("dot", t, row.D, planes)
    assert used == "dot_fast_c4planar", used
    return t, planes, out


def _dump_dot_rows(tile, path):
    """Run in a child process with SRCV_DOT_TILE_W set: the outputs of every dot row of `tile`."""
    out = {}
    for row in MATRIX:
        if row.kernel == "dot" and row.tile == tile:
            _, _, (cost, lowest, _, _) = run_dot_row(row)
            out[row.id] = (cost.cpu(), lowest.cpu())
    torch.save(out, path)


@pytest.mark.parametrize("row", [r for r in MATRIX if r.kernel == "dot" and r.tile == 16], ids=lambda r: r.id)
def test_dot_instantiation_vs_fp64_oracle(row):
    if process_tile() != 16:
        pytest.skip("this process runs the 32 x 1 warp tile")
    t, planes, (cost, lowest, planes_ret, mask) = run_dot_row(row)
    assert cost.shape == (row.B, row.D, row.H, row.W) and mask is None
    oc, _, op, _ = O.forward_dot(**t, num_depth_bins=row.D, depth_planes_bdhw=planes)
    t64, p64 = _fp64(t, planes)
    oc64, *_ = O.forward_dot(**t64, num_depth_bins=row.D, depth_planes_bdhw=p64)
    assert_cost_close("dot", cost, oc, oc64, what=row.id)
    if planes is None:
        assert torch.allclose(planes_ret[:, :, 0, 0].cpu(), op[:, :, 0, 0], rtol=3e-7, atol=0)
    assert_lowest_close("dot", lowest, planes_ret, oc, what=row.id)
    _argmax_is_lowest(cost, planes_ret, lowest)


@pytest.fixture(scope="module")
def tile32_outputs(tmp_path_factory):
    """The dot rows of warp tile 32, computed once in a child process started with SRCV_DOT_TILE_W=32."""
    path = tmp_path_factory.mktemp("tile32") / "dot_rows.pt"
    code = (f"import sys; sys.path.insert(0, {str(ROOT)!r}); "
            "from tests.test_gpu_instantiations import _dump_dot_rows; _dump_dot_rows(32, sys.argv[1])")
    env = dict(os.environ, SRCV_DOT_TILE_W="32")
    r = subprocess.run([sys.executable, "-c", code, str(path)], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-4000:]
    return torch.load(path)


@pytest.mark.parametrize("row", [r for r in MATRIX if r.kernel == "dot" and r.tile == 32], ids=lambda r: r.id)
def test_dot_tile32_instantiation_equals_tile16_bitwise(row, tile32_outputs):
    """The 32 x 1 warp tile against the 16 x 2 one on the same call: equal bit for bit, so the tile-16
    row's fp64 oracle check carries over."""
    if process_tile() != 16:
        pytest.skip("this process runs the 32 x 1 warp tile")
    cost32, lowest32 = tile32_outputs[row.id]
    _, _, (cost16, lowest16, _, _) = run_dot_row(replace(row, tile=16))
    assert torch.equal(cost32, cost16.cpu()), row.id
    assert torch.equal(lowest32, lowest16.cpu()), row.id


# --------------------------------------------------------------------------------------------- #
# wgmma metadata-MLP sweep                                                                       #
# --------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("row", [r for r in MATRIX if r.kernel == "hero"], ids=lambda r: r.id)
def test_hero_instantiation_vs_fp64_oracle(row):
    t, planes = row_inputs(row)
    sd = mlp_state(HERO_K, C, seed=_seed(row))
    (cost, lowest, planes_ret, mask), used = run("mlp", t, row.D, planes, sd)
    assert used == "mlp_tc_wgmma_f16x3", used
    assert cost.shape == (row.B, row.D, row.H, row.W) and mask.shape == (row.B, row.H, row.W)
    w = O.mlp_weights_from_state_dict(sd)
    oc, _, _, om = O.forward_mlp(**t, weights=w, num_depth_bins=row.D, depth_planes_bdhw=planes, return_mask=True)
    t64, p64 = _fp64(t, planes)
    oc64, *_ = O.forward_mlp(**t64, weights=tuple(x.double() for x in w), num_depth_bins=row.D,
                             depth_planes_bdhw=p64)
    assert_cost_close("mlp", cost, oc, oc64, what=row.id)
    assert_mask_close(mask, om, what=row.id)
    assert_lowest_close("mlp", lowest, planes_ret, oc, what=row.id)
    _argmax_is_lowest(cost, planes_ret, lowest)


def test_hero_128x96_two_frames_full_depth_properties():
    """The 512 x 384 frame size at the bench's plane count (cfg2's property checks at 128 x 96)."""
    B, D, H, W = 2, 64, 96, 128
    t = make_tuple(B, HERO_K, H, W, channels=C, seed=9601)
    sd = mlp_state(HERO_K, C, seed=9602)
    (cost, lowest, planes, mask), used = run("mlp", t, D, sd=sd)
    assert used == "mlp_tc_wgmma_f16x3" and cost.shape == (B, D, H, W)
    # shard invariance: frame 1 alone equals frame 1 inside the batch
    t1 = {k: (v[1:] if v.dim() > 0 and v.shape[0] == B else v) for k, v in t.items()}
    (cost1, lowest1, _, mask1), _ = run("mlp", t1, D, sd=sd)
    assert torch.equal(cost1, cost[1:]) and torch.equal(lowest1, lowest[1:]) and torch.equal(mask1, mask[1:])
    _argmax_is_lowest(cost, planes, lowest)
    # the fast manager class runs the same sweep; the fp32 SIMT variant agrees within the cost tolerance
    (cost_f, _, _, mask_f), _ = run("mlp", t, D, sd=sd, fast_cls=True)
    assert torch.equal(cost_f, cost) and torch.equal(mask_f, mask)
    (cost_g, _, _, mask_g), used_g = run("mlp", t, D, sd=sd, variant=_native.VARIANT_GENERIC)
    assert used_g == "mlp_generic_fp32" and torch.equal(mask_g, mask)
    err = (cost_g - cost).abs().max().item()
    assert err <= cost_tol("mlp", cost.cpu()), err
    # determinism
    (cost_r, lowest_r, _, mask_r), _ = run("mlp", t, D, sd=sd)
    assert torch.equal(cost_r, cost) and torch.equal(lowest_r, lowest) and torch.equal(mask_r, mask)


# --------------------------------------------------------------------------------------------- #
# per-pixel planes holding the per-plane values: the per-plane result, bit for bit               #
# --------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("kind,B,D,H,W", [
    *[("dot", B, D, H, W) for _, H, W in DOT_MAPS for B, D, _ in DOT_PLANES],
    *[("mlp", 1, 64, H, W) for _, H, W in HERO_MAPS],
])
def test_per_pixel_planes_equal_per_plane_bitwise(kind, B, D, H, W):
    """Both PER_PIXEL instantiations read the same plane value as the per-plane ones and run the same
    arithmetic on it, at every size and over the whole plane count."""
    t = make_tuple(B, HERO_K, H, W, channels=C, seed=7000 + H + D)
    sd = mlp_state(HERO_K, C, seed=7001) if kind == "mlp" else None
    (cost, lowest, planes, mask), _ = run(kind, t, D, sd=sd)
    assert planes.stride()[2:] == (0, 0)
    dense = planes.contiguous()                       # (B, D, H, W) tensor: the per-pixel path
    (cost_p, lowest_p, planes_p, mask_p), _ = run(kind, t, D, dense.cpu(), sd=sd)
    assert torch.equal(cost_p, cost) and torch.equal(lowest_p, lowest)
    if kind == "mlp":
        assert torch.equal(mask_p, mask)


# --------------------------------------------------------------------------------------------- #
# training path at the reference's default resolution                                           #
# --------------------------------------------------------------------------------------------- #
def test_dot_backward_at_96x128():
    """The backward kernel has no size specialisation, but at 96 x 128 its gradients sum ~3 000 tile
    partials per entry through atomics.  Against fp64 autograd through the oracle."""
    from tests.test_zzz_gpu_mlp_backward import _grad_close, _rel
    B, K, H, W, D = 2, 3, 96, 128, 8
    t = make_tuple(B, K, H, W, channels=C, seed=9611)
    gcost = torch.randn(B, D, H, W, generator=torch.Generator().manual_seed(9612))
    tc = {k: v.double() for k, v in t.items()}
    tc["cur_feats"] = tc["cur_feats"].clone().requires_grad_(True)
    tc["src_feats"] = tc["src_feats"].clone().requires_grad_(True)
    oc64, *_ = O.forward_dot(**tc, num_depth_bins=D)
    (oc64 * gcost.double()).sum().backward()
    d = to_device(t, "cuda")
    d["cur_feats"] = d["cur_feats"].clone().requires_grad_(True)
    d["src_feats"] = d["src_feats"].clone().requires_grad_(True)
    m = S.CostVolumeManager(H, W, num_depth_bins=D).cuda()
    cost, *_ = m(**d)
    (cost * gcost.cuda()).sum().backward()
    torch.cuda.synchronize()
    assert _native.last_variant() == "dot_backward_atomic"
    for name in ("cur_feats", "src_feats"):
        o, r = d[name].grad, tc[name].grad
        print(f"[grad] dot 96x128 {name}: max-rel {_rel(o, r):.2e}")
        assert _grad_close(o, r), f"grad {name}: rel err {_rel(o, r):.2e}"


def test_hero_backward_at_96x128():
    """Metadata-MLP training at 96 x 128: the weight gradients sum ~3 000 tile partials per entry."""
    from tests.test_zzz_gpu_mlp_backward import _grad_close, _oracle_grads, _rel
    B, H, W, D = 2, 96, 128, 8
    t = make_tuple(B, HERO_K, H, W, channels=C, seed=9621)
    gcost = torch.randn(B, D, H, W, generator=torch.Generator().manual_seed(9622))
    m = S.FeatureVolumeManager(H, W, num_depth_bins=D, mlp_channels=[0, 128, 128, 1], matching_dim_size=C,
                               num_source_views=HERO_K)
    m.load_state_dict({**m.state_dict(), **mlp_state(HERO_K, C, seed=9623)})
    m = m.cuda().train()
    d = to_device(t, "cuda")
    d["cur_feats"] = d["cur_feats"].clone().requires_grad_(True)
    d["src_feats"] = d["src_feats"].clone().requires_grad_(True)
    cost, *_ = m(**d)
    (cost * gcost.cuda()).sum().backward()
    torch.cuda.synchronize()
    assert _native.last_variant() == "mlp_backward_fp32_recompute"
    params = [p for i in (0, 2, 4) for p in (m.mlp.net[i].weight, m.mlp.net[i].bias)]
    _, ref = _oracle_grads(t, params, D, gcost, None)
    ours = [d["cur_feats"].grad, d["src_feats"].grad] + [p.grad for p in params]
    for name, o, r in zip(("cur", "src", "w1", "b1", "w2", "b2", "w3", "b3"), ours, ref):
        assert o is not None and tuple(o.shape) == tuple(r.shape), name
        print(f"[grad] hero 96x128 {name}: max-rel {_rel(o, r):.2e}")
        assert _grad_close(o, r), f"grad {name}: rel err {_rel(o, r):.2e}"
