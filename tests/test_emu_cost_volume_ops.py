"""The ``b200cv`` operator forwards and the managers' ``warp_features`` driven on the CPU against the
host-emulated C-ABI library (tests/emu): the operators and the managers share one launch per sweep,
so on the same planes they must return the same bits, and both ``warp_features`` methods take their
plane through the same dtype / device check."""
import contextlib
import types

import pytest
import torch

import simplerecon_b200 as S
from simplerecon_b200 import _native, cost_volume, torch_ops
from simplerecon_b200.synthetic import make_tuple, mlp_state
from tests import emu


@pytest.fixture()
def emulated(monkeypatch):
    """The device gate, the loaded library and the torch.cuda calls patched as in
    tests/test_emu_python_stack.py, so the product's Python code runs on CPU tensors."""
    lib = emu.load_or_skip()
    lib.emu_set_sms(4)
    lib.srcv_set_variant(_native.VARIANT_AUTO)
    monkeypatch.setattr(_native, "_lib", lib)
    monkeypatch.setattr(cost_volume, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: types.SimpleNamespace(cuda_stream=0))
    # CUDA allocations are >= 256-byte aligned (the C ABI requires it of the workspace); CPU ones are not
    real_empty = torch.empty

    def aligned_empty(*size, **kw):
        if kw.get("dtype") is torch.uint8 and len(size) == 1 and isinstance(size[0], int):
            buf = real_empty(size[0] + 256, **kw)
            off = (-buf.data_ptr()) % 256
            return buf[off:off + size[0]]
        return real_empty(*size, **kw)

    monkeypatch.setattr(torch, "empty", aligned_empty)
    return lib


@pytest.mark.parametrize("per_pixel", [False, True])
@pytest.mark.parametrize("kind", ["dot", "mlp"])
def test_operator_forward_equals_manager(emulated, kind, per_pixel):
    """``_dot_forward`` / ``_mlp_forward`` on ``(B,D)`` and ``(B,D,H,W)`` planes against the manager's
    ``forward`` given the same planes as ``depth_planes_bdhw``, at the hero shape (K=7, C=16, MLP
    128/128: the tensor-core sweep).  The operator packs the weight image into its workspace, the
    manager uses its cached image."""
    B, K, C, H, W, D = 2, 7, 16, 6, 16, 4
    t = make_tuple(B, K, H, W, channels=C, seed=51)
    g = torch.Generator().manual_seed(52)
    if per_pixel:
        planes = 0.3 + 4.0 * torch.rand(B, D, H, W, generator=g)
        planes_bdhw = planes
    else:
        planes = 0.3 + 4.0 * torch.rand(B, D, generator=g)
        planes_bdhw = planes.view(B, D, 1, 1).expand(B, D, H, W)
    cams = (t["src_extrinsics"], t["src_Ks"], t["cur_invK"])
    if kind == "dot":
        m = S.CostVolumeManager(H, W, num_depth_bins=D)
        cost, lowest = torch_ops._dot_forward(t["cur_feats"], t["src_feats"], *cams, planes)
    else:
        m = S.FeatureVolumeManager(H, W, num_depth_bins=D, mlp_channels=[0, 128, 128, 1], matching_dim_size=C,
                                   num_source_views=K)
        m.load_state_dict({**m.state_dict(), **mlp_state(views=K, channels=C, seed=1)})
        lin = [l for l in m.mlp.net if isinstance(l, torch.nn.Linear)]
        cost, lowest, mask = torch_ops._mlp_forward(
            t["cur_feats"], t["src_feats"], t["src_extrinsics"], t["src_poses"], t["src_Ks"], t["cur_invK"], planes,
            *[p.detach() for l in lin for p in (l.weight, l.bias)])
        assert _native.last_variant() == "mlp_tc_wgmma_f16x3"
    with torch.no_grad():
        cost_m, lowest_m, planes_m, mask_m = m(**t, depth_planes_bdhw=planes_bdhw, return_mask=True)
    assert planes_m is planes_bdhw and cost.shape == (B, D, H, W) and lowest.shape == (B, H, W)
    assert torch.equal(cost, cost_m) and torch.equal(lowest, lowest_m)
    if kind == "mlp":
        assert mask.dtype == torch.bool and torch.equal(mask, mask_m)


def _warp_args(B=1, K=2, C=8, H=9, W=12):
    t = make_tuple(B, K, H, W, channels=C, seed=15)
    return S.CostVolumeManager(H, W, num_depth_bins=4), (t["src_feats"].reshape(B * K, C, H, W), t["src_extrinsics"],
                                                         t["src_Ks"], t["cur_invK"]), (B, K, C, H, W)


def test_warp_features_upcasts_a_half_plane(emulated):
    """The base class's ``warp_features`` reads an fp16 plane as the fp32 plane of the same value, as
    the fast class does."""
    m, args, (B, K, C, H, W) = _warp_args()
    plane = torch.full((B, 1, 1, 1), 1.7, dtype=torch.float16).expand(B, 1, H, W)
    half = m.warp_features(*args, plane, B, K, C)
    full = m.warp_features(*args, plane.float(), B, K, C)
    assert half[2].shape == (B, K, C, H, W) and half[1].shape == half[3].shape == (B, K, H, W)
    for a, b in zip(half, full):
        assert torch.equal(a, b)


def test_warp_features_refuses_a_plane_on_another_device(emulated):
    m, args, (B, K, C, H, W) = _warp_args()
    plane = torch.full((B, 1, H, W), 1.7, device="meta")
    with pytest.raises(ValueError, match="is on meta"):
        m.warp_features(*args, plane, B, K, C)
