"""CPU: install(fusion=True, unbounded_fusion=True) — ``get_fuser`` for ``--depth_fuser ours`` without a ground-truth
mesh builds a SparseTSDF (DESIGN §4.16), with and without colour; with one, and with the flag off, the fusers are
exactly the ones built before; uninstall() restores everything.  Against stand-ins of the reference modules, as the
colour-fusion install tests use."""
import importlib
import sys
import types

import pytest

from simplerecon_b200 import fusers, tsdf as tsdf_mod

install_mod = importlib.import_module("simplerecon_b200.install")


def _fake_reference(monkeypatch):
    ref_tsdf = types.ModuleType("tools.tsdf")
    ref_tsdf.TSDF, ref_tsdf.TSDFFuser = type("TSDF", (), {}), type("TSDFFuser", (), {})
    fh = types.ModuleType("tools.fusers_helper")
    fh.TSDF, fh.TSDFFuser = ref_tsdf.TSDF, ref_tsdf.TSDFFuser
    fh.calls = []
    fh.get_fuser = lambda opts, scan: fh.calls.append((opts, scan)) or "original"
    fh.ScannetDataset = types.SimpleNamespace(get_gt_mesh_path=lambda root, split, scan: f"{root}/{split}/{scan}.ply")
    tools = types.ModuleType("tools")
    tools.tsdf, tools.fusers_helper = ref_tsdf, fh
    cv = types.ModuleType("modules.cost_volume")
    modules = types.ModuleType("modules")
    modules.cost_volume = cv
    for name, mod in {"tools": tools, "tools.tsdf": ref_tsdf, "tools.fusers_helper": fh, "modules": modules,
                      "modules.cost_volume": cv}.items():
        monkeypatch.setitem(sys.modules, name, mod)
    return ref_tsdf, fh


def _opts(**kw):
    base = dict(dataset="arkit", dataset_path="/data", split="test", depth_fuser="ours", fuse_color=False,
                fusion_resolution=0.02, fusion_max_depth=3.0)
    return types.SimpleNamespace(**{**base, **kw})


@pytest.mark.parametrize("with_color_flag", [False, True])
def test_unbounded_fusion_routes_ours_without_gt_to_sparse(monkeypatch, with_color_flag):
    ref_tsdf, fh = _fake_reference(monkeypatch)
    orig = fh.get_fuser
    made = []
    monkeypatch.setattr(fusers, "ColorFuser", lambda **kw: made.append(kw) or "color")
    with pytest.raises(ValueError, match="fusion=True"):
        install_mod.install(unbounded_fusion=True)
    try:
        install_mod.install(fusion=True, fuse_color=with_color_flag, unbounded_fusion=True)
        assert fh.get_fuser is not orig and fh.TSDF is tsdf_mod.TSDF and ref_tsdf.TSDFFuser is tsdf_mod.TSDFFuser
        # no ground-truth mesh (every dataset but ScanNet): the sparse volume, with colour when asked and installed
        for fuse_color in (False, True):
            assert fh.get_fuser(_opts(fuse_color=fuse_color), "scan") == "color"
            assert made[-1] == dict(gt_path=None, fusion_resolution=0.02, max_fusion_depth=3.0,
                                    fuse_color=fuse_color and with_color_flag, unbounded=True)
        # a ground-truth mesh: the dense path as before (ColorFuser with colour and its flag, else the original)
        n = len(made)
        o = _opts(dataset="scannet")
        assert fh.get_fuser(o, "scene0707_00") == "original" and fh.calls[-1] == (o, "scene0707_00")
        if with_color_flag:
            assert fh.get_fuser(_opts(dataset="scannet", fuse_color=True), "scene0707_00") == "color"
            assert made[-1] == dict(gt_path="/data/test/scene0707_00.ply", fusion_resolution=0.02,
                                    max_fusion_depth=3.0, fuse_color=True)
        assert len(made) == n + int(with_color_flag)
        for kw in (dict(depth_fuser="open3d"), dict(depth_fuser="open3d", fuse_color=True), dict(depth_fuser="nope")):
            o = _opts(**kw)
            assert fh.get_fuser(o, "s") == "original" and fh.calls[-1] == (o, "s")
    finally:
        install_mod.uninstall()
    assert fh.get_fuser is orig and fh.TSDF is not tsdf_mod.TSDF


def test_flag_off_is_todays_install(monkeypatch):
    _, fh = _fake_reference(monkeypatch)
    orig = fh.get_fuser
    try:
        install_mod.install(fusion=True)
        assert fh.get_fuser is orig
    finally:
        install_mod.uninstall()
    try:
        install_mod.install(fusion=True, fuse_color=True)
        made = []
        monkeypatch.setattr(fusers, "ColorFuser", lambda **kw: made.append(kw) or "color")
        assert fh.get_fuser(_opts(fuse_color=True), "s") == "color"
        assert made == [dict(gt_path=None, fusion_resolution=0.02, max_fusion_depth=3.0, fuse_color=True)]
        assert fh.get_fuser(_opts(), "s") == "original"
    finally:
        install_mod.uninstall()
    assert fh.get_fuser is orig


def test_color_fuser_builds_the_sparse_volume(monkeypatch):
    """ColorFuser(unbounded=True) without a mesh: a SparseTSDF on the ±10 m cube's lattice (no device needed to
    check what is built: the constructor is recorded)."""
    built = []
    monkeypatch.setattr(fusers, "SparseTSDF", lambda voxel, max_blocks, color: built.append((voxel, max_blocks, color))
                        or types.SimpleNamespace(voxel_size=voxel))
    f = fusers.ColorFuser(gt_path=None, fusion_resolution=0.02, fuse_color=False, unbounded=True, max_blocks=1000)
    assert built == [(0.02, 1000, False)] and f.tsdf_fuser_pred.max_depth == 3
    fusers.ColorFuser(gt_path=None, fusion_resolution=0.04, unbounded=True)
    assert built[-1] == (0.04, 1 << 17, True)
