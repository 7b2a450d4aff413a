"""CPU tier for the sweep kernels' compile-time instantiations (see tests/test_gpu_instantiations.py).

* A coverage guard: the dispatch lists of csrc/srcv_dot.cu and csrc/srcv_mlp_tc.cu are parsed, and
  every (kernel, map size, planes mode, warp tile) they instantiate must have a row in the GPU matrix
  whose shape really reaches it.  Adding an instantiation without a test fails here.
* The dot rows of that matrix at 128 x 96 and 64 x 48 on the host emulation (tests/emu), with 132 SMs
  as on an H100 SXM so that the plane-loop split is the one the GPU takes, against the oracle's fp64
  evaluation; the 32 x 1 warp tile in a child process (the tile is latched on the first call), equal
  to the 16 x 2 tile bit for bit.
* Per-pixel planes holding the per-plane values give the per-plane result bit for bit, for both kernels.
* Behind SRCV_EMU_SLOW (about a minute per case): the wgmma kernel's 128 x 96 instantiations with range
  and per-pixel planes, D = 2 and D = 3, against fp64.
"""
from __future__ import annotations

import functools
import os
import re
import subprocess
import sys
from dataclasses import replace
from pathlib import Path

import pytest
import torch

from oracle import costvolume_oracle as O
from simplerecon_b200 import _native as N
from simplerecon_b200.synthetic import make_tuple, mlp_state
from tests import emu
from tests.parity import assert_cost_close, assert_lowest_close, assert_mask_close
from tests.test_gpu_instantiations import DOT_WARPS_PER_SM, MATRIX, C, dot_plane_split, row_inputs

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "simplerecon_b200" / "csrc"
H100_SMS = 132
SLOW = pytest.mark.skipif(not os.environ.get("SRCV_EMU_SLOW"), reason="about a minute per case: set SRCV_EMU_SLOW=1")


# --------------------------------------------------------------------------------------------- #
# coverage guard                                                                                 #
# --------------------------------------------------------------------------------------------- #
def dispatched_instantiations():
    """{(kernel, (TW, TH), per_pixel, tile)} as the launchers instantiate them, and the sized lists
    (W, H) in dispatch order."""
    dot = (CSRC / "srcv_dot.cu").read_text()
    tc = (CSRC / "srcv_mlp_tc.cu").read_text()
    dot_sizes = [(int(w), int(h)) for w, h in re.findall(r"^\s*SRCV_SIZED\((\d+),\s*(\d+)\)", dot, re.M)]
    assert re.search(r"dot_fast_kernel<PER_PIXEL,\s*0,\s*0,\s*kTileW>", dot), "run-time-size dot launch not found"
    dot_modes = {(pp == "true", int(tile)) for pp, tile in re.findall(r"launch_fast_sized<(true|false),\s*(\d+)>", dot)}
    tile_env = re.search(r'getenv\("SRCV_DOT_TILE_W"\).*?\n.*?atoi\(e\)\s*==\s*(\d+)\)\s*\?\s*(\d+)\s*:\s*(\d+)', dot)
    assert tile_env, "SRCV_DOT_TILE_W parsing not found"
    assert {int(tile_env.group(2)), int(tile_env.group(3))} == {tile for _, tile in dot_modes}
    tc_sizes = [(int(w), int(h)) for w, h in re.findall(r"SRCV_TC_LAUNCH\(PP,\s*(\d+),\s*(\d+)\)", tc)]
    tc_modes = {pp == "true" for pp in re.findall(r"SRCV_TC_SIZES\((true|false)\)", tc)}
    assert dot_sizes and (0, 0) in tc_sizes and dot_modes and tc_modes == {False, True}
    want = {("dot", size, pp, tile) for size in [*dot_sizes, (0, 0)] for pp, tile in dot_modes}
    want |= {("hero", size, pp, 0) for size in tc_sizes for pp in tc_modes}
    return want, {"dot": dot_sizes, "hero": [s for s in tc_sizes if s != (0, 0)]}


def test_gpu_matrix_covers_every_dispatched_instantiation():
    want, sized = dispatched_instantiations()
    have = {(r.kernel, r.inst, r.per_pixel, r.tile) for r in MATRIX}
    missing = sorted(want - have)
    assert not missing, f"instantiations without a row in tests/test_gpu_instantiations.py MATRIX: {missing}"
    assert not sorted(have - want), f"MATRIX rows for instantiations the launchers do not have: {sorted(have - want)}"
    for r in MATRIX:
        # the row's map size reaches the instantiation it names
        reached = (r.W, r.H) if (r.W, r.H) in sized[r.kernel] else (0, 0)
        assert reached == r.inst, f"{r.id}: a {r.H}x{r.W} map runs the {reached} instantiation"
        if r.kernel == "dot":
            # both argmax forms at every instantiation, and the row's shape reaches the form it names
            assert (dot_plane_split(r.B, r.D, r.H, r.W, r.tile, H100_SMS) > 1) == r.split, r.id
    for key in want:
        if key[0] == "dot":
            forms = {r.split for r in MATRIX if (r.kernel, r.inst, r.per_pixel, r.tile) == key}
            assert forms == {False, True}, f"{key}: fused and split argmax not both covered"
        else:
            ds = {r.D % 2 for r in MATRIX if (r.kernel, r.inst, r.per_pixel, r.tile) == key}
            assert ds == {0, 1}, f"{key}: even and odd D not both covered"


# --------------------------------------------------------------------------------------------- #
# dot rows on the emulation                                                                      #
# --------------------------------------------------------------------------------------------- #
EMU_DOT_SIZES = {(128, 96), (64, 48)}
EMU_DOT_ROWS = [r for r in MATRIX if r.kernel == "dot" and r.inst in EMU_DOT_SIZES]


@pytest.fixture(scope="module")
def lib():
    lib = emu.load_or_skip()
    yield lib
    lib.emu_set_sms(4)
    lib.srcv_set_variant(N.VARIANT_AUTO)


def _process_tile():
    return 32 if os.environ.get("SRCV_DOT_TILE_W", "").strip() == "32" else 16


@functools.lru_cache(maxsize=None)
def emu_dot_row(row):
    """(cost, lowest, planes) of a dot row on the emulated C ABI with the H100's SM count."""
    assert row.tile == _process_tile(), f"{row.id}: this process runs warp tile {_process_tile()}"
    lib = emu.load()
    lib.emu_set_sms(H100_SMS)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    if "SRCV_DOT_WARPS_PER_SM" not in os.environ:
        assert (dot_plane_split(row.B, row.D, row.H, row.W, row.tile, H100_SMS, DOT_WARPS_PER_SM) > 1) == row.split
    t, planes = row_inputs(row)
    cost, lowest, planes_bd, used = emu.dot_forward(t, row.D, planes=planes)
    assert used == "dot_fast_c4planar", used
    return cost, lowest, planes if planes is not None else planes_bd.view(row.B, row.D, 1, 1)


def _dump_emu_dot_rows(tile, path):
    """Run in a child process with SRCV_DOT_TILE_W set."""
    torch.save({r.id: emu_dot_row(r)[:2] for r in EMU_DOT_ROWS if r.tile == tile}, path)


@pytest.mark.parametrize("row", [r for r in EMU_DOT_ROWS if r.tile == 16], ids=lambda r: r.id)
def test_emu_dot_instantiation_vs_fp64_oracle(lib, row):
    if _process_tile() != 16:
        pytest.skip("this process runs the 32 x 1 warp tile")
    cost, lowest, planes = emu_dot_row(row)
    t, pp = row_inputs(row)
    oc, *_ = O.forward_dot(**t, num_depth_bins=row.D, depth_planes_bdhw=pp)
    oc64, *_ = O.forward_dot(**{k: v.double() for k, v in t.items()}, num_depth_bins=row.D,
                             depth_planes_bdhw=None if pp is None else pp.double())
    assert_cost_close("dot", cost, oc, oc64, what=f"emu {row.id}")
    assert_lowest_close("dot", lowest, planes, oc, what=f"emu {row.id}")
    idx = cost.argmax(1, keepdim=True)
    assert torch.equal(torch.gather(planes.expand_as(cost), 1, idx).squeeze(1), lowest)
    if not row.per_pixel:
        # the PER_PIXEL instantiation on per-pixel planes holding these values: the same bits
        c2, l2, _, _ = emu.dot_forward(t, row.D, planes=planes.expand_as(cost).contiguous())
        assert torch.equal(c2, cost) and torch.equal(l2, lowest)


def test_emu_dot_tile32_equals_tile16_bitwise(lib, tmp_path):
    if _process_tile() != 16:
        pytest.skip("this process runs the 32 x 1 warp tile")
    path = tmp_path / "dot_tile32.pt"
    code = (f"import sys; sys.path.insert(0, {str(ROOT)!r}); "
            "from tests.test_emu_instantiations import _dump_emu_dot_rows; _dump_emu_dot_rows(32, sys.argv[1])")
    r = subprocess.run([sys.executable, "-c", code, str(path)], cwd=ROOT, capture_output=True, text=True,
                       env=dict(os.environ, SRCV_DOT_TILE_W="32"), timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    got = torch.load(path)
    rows32 = [r for r in EMU_DOT_ROWS if r.tile == 32]
    assert sorted(got) == sorted(r.id for r in rows32)
    for row in rows32:
        cost16, lowest16, _ = emu_dot_row(replace(row, tile=16))
        cost32, lowest32 = got[row.id]
        assert torch.equal(cost32, cost16) and torch.equal(lowest32, lowest16), row.id


# --------------------------------------------------------------------------------------------- #
# wgmma kernel                                                                                   #
# --------------------------------------------------------------------------------------------- #
def _hero_weights(seed):
    sd = mlp_state(7, C, seed=seed)
    return [sd[f"mlp.net.{i}.{n}"].clone() for i in (0, 2, 4) for n in ("weight", "bias")]


def _hero_per_pixel_equals_range(t, D, wts):
    cost, lowest, planes_bd, mask, used = emu.mlp_forward(t, D, wts)
    assert used == "mlp_tc_wgmma_f16x3", used
    B, _, H, W = cost.shape
    dense = planes_bd.view(B, D, 1, 1).expand(B, D, H, W).contiguous()
    c2, l2, _, m2, _ = emu.mlp_forward(t, D, wts, planes=dense)
    assert torch.equal(c2, cost) and torch.equal(l2, lowest) and torch.equal(m2, mask)


@pytest.mark.parametrize("D", [4, 5])
def test_emu_hero_per_pixel_planes_equal_range_bitwise(lib, D):
    """The run-time-size pair of wgmma instantiations, a ragged 9 x 21 map (the compile-time sizes
    take a minute each here: test_emu_hero_128x96 below)."""
    lib.emu_set_sms(3)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    _hero_per_pixel_equals_range(make_tuple(1, 7, 9, 21, channels=C, seed=9630 + D), D, _hero_weights(9631))


@SLOW
@pytest.mark.parametrize("D", [2, 3])
@pytest.mark.parametrize("per_pixel", [False, True])
def test_emu_hero_128x96(lib, per_pixel, D):
    """mlp_tc_kernel<PER_PIXEL, 128, 96> on one 512 x 384 frame.  At this size the oracle's own fp32
    result is ~9e-6 from its fp64 evaluation, the kernel ~2.5e-6: judged against fp64."""
    lib.emu_set_sms(8)
    lib.srcv_set_variant(N.VARIANT_AUTO)
    B, H, W = 1, 96, 128
    t = make_tuple(B, 7, H, W, channels=C, seed=9640 + D)
    wts = _hero_weights(9641)
    planes = (0.3 + 4.0 * torch.rand(B, D, H, W, generator=torch.Generator().manual_seed(9642))) if per_pixel else None
    cost, lowest, planes_bd, mask, used = emu.mlp_forward(t, D, wts, planes=planes)
    assert used == "mlp_tc_wgmma_f16x3", used
    oc, _, _, om = O.forward_mlp(**t, weights=tuple(wts), num_depth_bins=D, depth_planes_bdhw=planes, return_mask=True)
    o64, *_ = O.forward_mlp(**{k: v.double() for k, v in t.items()}, weights=tuple(w.double() for w in wts),
                            num_depth_bins=D, depth_planes_bdhw=None if planes is None else planes.double())
    assert_cost_close("mlp", cost, oc, o64, what=f"emu wgmma 128x96 D={D} per_pixel={per_pixel}")
    assert_mask_close(mask, om, what="emu wgmma 128x96")
    pl = planes if per_pixel else planes_bd.view(B, D, 1, 1)
    assert_lowest_close("mlp", lowest, pl, oc, what="emu wgmma 128x96")
    if not per_pixel:
        dense = planes_bd.view(B, D, 1, 1).expand(B, D, H, W).contiguous()
        c2, l2, _, m2, _ = emu.mlp_forward(t, D, wts, planes=dense)
        assert torch.equal(c2, cost) and torch.equal(l2, lowest) and torch.equal(m2, mask)
