"""CPU: the depth-metrics kernels (csrc/srcv_metrics.cuh) compiled for the host (tests/emu), through the C ABI
and simplerecon_b200.metrics, against the oracle's fp32-terms / fp64-sums mode (oracle/metrics_oracle.py):
counts and a-metrics exact, continuous metrics within 1e-6 relative with NaN and inf in the same places;
the resampled prediction against F.interpolate (nearest bit-equal, bilinear within 2 ulp); determinism;
argument checks; and install(metrics=True)."""
import contextlib
import ctypes as C
import importlib.util
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

import simplerecon_b200 as S
from oracle import metrics_oracle as M
from oracle.ref_import import reference_available, reference_root
from simplerecon_b200 import _native, metrics as SM
from tests import emu
from tests.test_metrics_oracle_vs_reference import make_batched_inputs, make_flat_inputs


@pytest.fixture()
def emulated(monkeypatch):
    lib = emu.load_or_skip()
    monkeypatch.setattr(_native, "_lib", lib)
    monkeypatch.setattr(SM, "_require_cuda", lambda t: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: types.SimpleNamespace(cuda_stream=0))
    real_empty = torch.empty

    def aligned_empty(*size, **kw):
        if kw.get("dtype") is torch.uint8 and len(size) == 1 and isinstance(size[0], int):
            buf = real_empty(size[0] + 256, **kw)
            off = (-buf.data_ptr()) % 256
            return buf[off:off + size[0]]
        return real_empty(*size, **kw)

    monkeypatch.setattr(torch, "empty", aligned_empty)
    return lib


def ulp_diff(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return (a.float().contiguous().view(torch.int32).long() - b.float().contiguous().view(torch.int32).long()).abs()


def check_metrics(metrics, counts, gt_bN, pred_bN, valid_bN=None, flat=False, mult_a=False):
    """kernel (B,12) / (B,) against the fp64-sum oracle on the same (B, N) inputs"""
    om, oc = M.metrics_fp64(gt_bN.cpu().float(), pred_bN.cpu().float(),
                            None if valid_bN is None else valid_bN.cpu(), flat=flat, mult_a=mult_a)
    m = metrics.cpu()
    assert m.dtype == torch.float32 and m.shape == om.shape
    assert torch.equal(counts.cpu(), oc), (counts, oc)
    a, oa = m[:, 5:], om[:, 5:]
    assert torch.equal(a.isnan(), oa.isnan()) and torch.equal(a[~a.isnan()], oa[~oa.isnan()]), (a, oa)
    c, occ = m[:, :5], om[:, :5]
    assert torch.equal(c.isnan(), occ.isnan()), (c, occ)
    assert torch.equal(c.isinf(), occ.isinf()) and torch.equal(c[c.isinf()], occ[occ.isinf()])
    fin = torch.isfinite(occ)
    assert ((c[fin].double() - occ[fin].double()).abs() <= 1e-6 * occ[fin].double().abs()).all(), (c, occ)
    return om


# ---- the reference's two functions -------------------------------------------------------------

@pytest.mark.parametrize("seed,mult_a", [(0, False), (1, True), (2, False)])
def test_batched_edge_cases(emulated, seed, mult_a):
    gt, pred, valid = make_batched_inputs(seed)
    d = S.compute_depth_metrics_batched(gt, pred, valid, mult_a=mult_a)
    assert list(d) == list(M.KEYS) and all(v.shape == (gt.shape[0],) for v in d.values())
    base = d["abs_diff"]._base
    assert base is not None and all(v._base is base for v in d.values())        # views of one result
    metrics = torch.stack(list(d.values()), 1)
    check_metrics(metrics, valid.sum(1), gt, pred, valid, mult_a=mult_a)
    ref32 = M.compute_depth_metrics_batched(gt, pred, valid, mult_a=mult_a)     # a-metrics: the reference's bits
    for k in M.KEYS[5:]:
        torch.testing.assert_close(d[k], ref32[k], rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("case", ["finite", "finite_mult_a", "nan", "empty", "edges"])
def test_flat_cases(emulated, case):
    gt, pred, mult_a = make_flat_inputs(case)
    d = S.compute_depth_metrics(gt, pred, mult_a=mult_a)
    assert list(d) == list(M.KEYS) and all(v.dim() == 0 for v in d.values())
    check_metrics(torch.stack(list(d.values()))[None], torch.tensor([gt.numel()]), gt[None], pred[None], flat=True,
                  mult_a=mult_a)
    ref32 = M.compute_depth_metrics(gt, pred, mult_a=mult_a)
    for k in M.KEYS:
        if k in M.KEYS[5:] or case == "empty":
            torch.testing.assert_close(d[k], ref32[k], rtol=0, atol=0, equal_nan=True)
        else:
            torch.testing.assert_close(d[k], ref32[k], rtol=2e-6, atol=0, equal_nan=True)


def test_flat_nan_and_batched_nanmean_differ(emulated):
    """pred = -1: log is NaN; the flat metrics make rmse_log NaN, the batched ones drop the pixel. pred = 0: inf."""
    gt = torch.tensor([[2.0, 3.0, 1.5, 4.0]])
    for p, flat_log in ((-1.0, "nan"), (0.0, "inf")):
        pred = torch.tensor([[2.2, 2.5, p, 4.0]])
        f = S.compute_depth_metrics(gt[0], pred[0])
        b = S.compute_depth_metrics_batched(gt, pred, torch.ones_like(gt, dtype=torch.bool))
        assert (f["rmse_log"].isnan() if flat_log == "nan" else f["rmse_log"].isinf())
        assert torch.isfinite(b["rmse_log"]).all() if p < 0 else b["rmse_log"].isinf().all()
        assert f["a25"].item() == b["a25"].item() == (1.0 if p < 0 else 0.75)     # negative counts as accurate, zero not


def test_half_inputs_are_upcast(emulated):
    gt, pred, valid = make_batched_inputs(3)
    keep = torch.isfinite(gt) & torch.isfinite(pred) & (pred.abs() < 6e4)
    gh, ph = gt.where(keep, 1.0).half(), pred.where(keep, 1.0).half()
    d = S.compute_depth_metrics_batched(gh, ph, valid)
    assert d["abs_rel"].dtype == torch.float16 and d["a5"].dtype == torch.float32   # the reference's result dtypes
    om, _ = M.metrics_fp64(gh.float(), ph.float(), valid)
    torch.testing.assert_close(d["a5"], om[:, 5], rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(d["abs_rel"], om[:, 1].half(), rtol=0, atol=0, equal_nan=True)
    db = S.compute_depth_metrics(gt[0][keep[0]].bfloat16(), pred[0][keep[0]].bfloat16())
    assert db["rmse"].dtype == torch.bfloat16 and db["a1"].dtype == torch.float32


# ---- depth_metrics: the prediction sampled on the ground-truth grid ----------------------------

def _depth_batch(seed, B, H, W, Hp, Wp, empty=()):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(B, 1, H, W, generator=g) * 5
    pred = torch.rand(B, 1, Hp, Wp, generator=g) * 5 + 0.05
    gt[:, :, ::5, ::3] = 0.0                                  # holes below any validity threshold
    for b in empty:
        gt[b] = 0.3
    return gt, pred


def _resampled(pred, H, W, mode):
    if mode == "nearest":
        return F.interpolate(pred, size=(H, W), mode="nearest")
    return F.interpolate(pred, size=(H, W), mode="bilinear", align_corners=False)


@pytest.mark.parametrize("seed,B,H,W,Hp,Wp,mode,source,mult_a", [
    (0, 3, 24, 32, 12, 16, "nearest", "min_depth", True),          # test.py: 2x nearest, gt > 0.5, mult_a
    (1, 2, 17, 23, 7, 9, "nearest", "mask", False),                # ragged ratio
    (2, 2, 17, 23, 7, 9, "bilinear", "min_depth", False),
    (3, 16, 9, 11, 4, 5, "nearest", "min_depth", True),            # B = 16 with empty frames
    (4, 2, 13, 15, 40, 50, "nearest", "all", False),               # prediction larger than the ground truth
    (5, 2, 13, 15, 40, 50, "bilinear", "mask", False),
    (6, 2, 19, 21, 19, 21, "bilinear", "min_depth", False),        # same size: identity
    (7, 1, 40, 37, 20, 14, "bilinear", "all", True),
])
def test_depth_metrics_matrix(emulated, seed, B, H, W, Hp, Wp, mode, source, mult_a):
    gt, pred = _depth_batch(seed, B, H, W, Hp, Wp, empty=(1, 4, 9) if B == 16 else ())
    valid = {"mask": torch.rand(B, 1, H, W, generator=torch.Generator().manual_seed(seed)) > 0.4,
             "min_depth": gt > 0.5, "all": torch.ones_like(gt, dtype=torch.bool)}[source]
    kw = {"mask": dict(valid_mask_b1hw=valid), "min_depth": dict(min_valid_depth=0.5), "all": {}}[source]
    metrics, counts, up = S.depth_metrics(gt, pred, mode=mode, mult_a=mult_a, return_upsampled=True, **kw)
    assert up.shape == gt.shape and counts.dtype == torch.int64
    ref_up = _resampled(pred, H, W, mode)
    if mode == "nearest":
        assert torch.equal(up, ref_up)
    else:
        assert ulp_diff(up, ref_up).max().item() <= 2
        assert torch.equal(up, M.resample_bilinear(pred, H, W))     # the oracle restates the kernel's FMAs
    om = check_metrics(metrics, valid.flatten(1).sum(1), gt.flatten(1), up.flatten(1), valid.flatten(1), mult_a=mult_a)
    if B == 16:
        assert (counts[[1, 4, 9]] == 0).all() and om[[1, 4, 9]].isnan().all() and metrics[[1, 4, 9]].isnan().all()
    m2, c2 = S.depth_metrics(gt, pred, mode=mode, mult_a=mult_a, **kw)  # without the resampled output; same bits
    assert torch.equal(m2.view(torch.int32), metrics.view(torch.int32)) and torch.equal(c2, counts)


def test_nearest_index_rule_matches_interpolate_at_the_test_shape(emulated):
    """192x256 -> 480x640 (test.py's shapes): the oracle's index rule and the kernel are F.interpolate's bits"""
    pred = torch.rand(1, 1, 192, 256, generator=torch.Generator().manual_seed(0)) + 0.1
    assert torch.equal(M.resample_nearest(pred, 480, 640), F.interpolate(pred, size=(480, 640), mode="nearest"))
    assert ulp_diff(M.resample_bilinear(pred, 480, 640), _resampled(pred, 480, 640, "bilinear")).max() <= 2


def test_runs_are_bit_identical(emulated):
    gt, pred = _depth_batch(11, 3, 33, 41, 12, 17)
    a = S.depth_metrics(gt, pred, min_valid_depth=0.5, mode="bilinear")
    b = S.depth_metrics(gt, pred, min_valid_depth=0.5, mode="bilinear")
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])


def test_python_argument_checks(emulated):
    gt, pred = _depth_batch(12, 2, 8, 10, 4, 5)
    with pytest.raises(ValueError):
        S.depth_metrics(gt, pred[:1])
    with pytest.raises(ValueError):
        S.depth_metrics(gt, pred, mode="bicubic")
    with pytest.raises(ValueError):
        S.depth_metrics(gt, pred, valid_mask_b1hw=gt > 0.5, min_valid_depth=0.5)
    with pytest.raises(ValueError):
        S.compute_depth_metrics(gt.flatten(), pred.flatten())
    with pytest.raises(ValueError):
        S.compute_depth_metrics_batched(gt.flatten(1), gt.flatten(1), (gt > 1).flatten(1)[:, :-1])
    with pytest.raises(ValueError):
        S.compute_depth_metrics(gt.double(), gt.double())
    with pytest.raises(ValueError):
        S.compute_depth_metrics(gt, gt.to("meta"))


def test_cpu_tensors_are_refused():
    with pytest.raises(RuntimeError):
        S.compute_depth_metrics(torch.ones(4), torch.ones(4))


# ---- the C ABI's host checks -------------------------------------------------------------------

def test_c_abi_argument_validation(emulated):
    lib = emulated
    gt, pred = torch.rand(2, 6, 7) + 0.1, torch.rand(2, 3, 4) + 0.1
    mask = torch.ones(2, 6, 7, dtype=torch.uint8)
    metrics, counts = torch.empty(2, 12), torch.empty(2, dtype=torch.int64)

    def args(**kw):
        a = dict(gt=gt.data_ptr(), pred=pred.data_ptr(), valid=mask.data_ptr(), min_valid_depth=0.5, B=2, H=6, W=7,
                 Hp=3, Wp=4, resample=_native.RESAMPLE_NEAREST, nan_mode=_native.METRICS_BATCHED,
                 valid_source=_native.METRICS_VALID_MASK, mult_a=0)
        a.update(kw)
        return _native.MetricsArgs(**a)

    def call(a, ws_bytes=None, m=metrics, c=counts):
        n = lib.srcv_metrics_workspace_bytes(C.byref(a))
        ws = emu.Call.workspace(None, max(n, 256))
        return lib.srcv_depth_metrics_f32(C.byref(a), C.c_void_p(m.data_ptr() if m is not None else 0),
                                          C.c_void_p(c.data_ptr() if c is not None else 0), None,
                                          C.c_void_p(ws.data_ptr()), n if ws_bytes is None else ws_bytes, None)

    assert call(args()) == 0
    assert counts.tolist() == [42, 42]
    assert lib.srcv_depth_metrics_f32(None, None, None, None, None, 0, None) == 1
    assert call(args(gt=None)) == 1 and call(args(valid=None)) == 1
    assert call(args(), m=None) == 1 and call(args(), c=None) == 1
    assert call(args(valid=None, valid_source=_native.METRICS_VALID_ALL)) == 0
    assert call(args(B=0)) == 2 and call(args(H=-1)) == 2 and call(args(B=70000)) == 2
    assert call(args(H=1 << 16, W=1 << 15)) == 2                                   # 2^31 pixels per frame
    assert call(args(resample=_native.RESAMPLE_IDENTITY)) == 2                      # sizes differ
    assert call(args(Hp=0)) == 2                                                    # nothing to resample
    assert call(args(resample=7)) == 4 and call(args(nan_mode=2)) == 4 and call(args(valid_source=3)) == 4
    assert call(args(), ws_bytes=16) == 3                                           # short workspace
    assert lib.srcv_metrics_workspace_bytes(C.byref(args(B=0))) == 0
    assert lib.srcv_metrics_workspace_bytes(C.byref(args(H=4096, W=4096))) == 2 * 16384 * 128


# ---- install(metrics=True) ---------------------------------------------------------------------

def _metrics_modules(monkeypatch, metrics_utils=None):
    """modules.cost_volume (install() always patches it) and utils.metrics_utils under their import names:
    the real reference module when given, else a stand-in holding the oracle's fp32 restatement."""
    pkg, cv, upkg = (types.ModuleType(n) for n in ("modules", "modules.cost_volume", "utils"))
    pkg.cost_volume = cv
    for n in ("CostVolumeManager", "FeatureVolumeManager", "FastFeatureVolumeManager"):
        setattr(cv, n, type(n, (torch.nn.Module,), {}))
    if metrics_utils is None:
        metrics_utils = types.ModuleType("utils.metrics_utils")
        metrics_utils.compute_depth_metrics = M.compute_depth_metrics
        metrics_utils.compute_depth_metrics_batched = M.compute_depth_metrics_batched
    upkg.metrics_utils = metrics_utils
    for name, mod in (("modules", pkg), ("modules.cost_volume", cv), ("utils", upkg),
                      ("utils.metrics_utils", metrics_utils)):
        monkeypatch.setitem(sys.modules, name, mod)
    monkeypatch.delitem(sys.modules, "experiment_modules.depth_model", raising=False)
    return metrics_utils


def check_install(monkeypatch, mu):
    """CPU calls through the installed functions return the original's bits; uninstall() restores both modules"""
    orig = (mu.compute_depth_metrics, mu.compute_depth_metrics_batched)
    gt, pred, valid = make_batched_inputs(4)
    want_b = orig[1](gt, pred, valid, mult_a=True)
    want_f = orig[0](gt[0][valid[0]], pred[0][valid[0]])
    dm = types.ModuleType("experiment_modules.depth_model")            # binds the name at import (:16)
    dm.compute_depth_metrics = mu.compute_depth_metrics
    monkeypatch.setitem(sys.modules, "experiment_modules.depth_model", dm)
    try:
        patched = S.install(metrics=True)
        assert mu.__name__ in patched and "experiment_modules.depth_model" in patched
        assert mu.compute_depth_metrics is not orig[0] and dm.compute_depth_metrics.__wrapped__ is orig[0]
        assert mu.compute_depth_metrics_batched.__wrapped__ is orig[1]
        got_b = mu.compute_depth_metrics_batched(gt, pred, valid, mult_a=True)
        got_f = dm.compute_depth_metrics(gt[0][valid[0]], pred[0][valid[0]])
        for want, got in ((want_b, got_b), (want_f, got_f)):
            assert list(got) == list(want)
            for k in want:
                torch.testing.assert_close(got[k], want[k], rtol=0, atol=0, equal_nan=True)
    finally:
        S.uninstall()
    assert (mu.compute_depth_metrics, mu.compute_depth_metrics_batched) == orig
    assert dm.compute_depth_metrics is orig[0]


def test_install_metrics_on_a_stand_in_module(monkeypatch):
    check_install(monkeypatch, _metrics_modules(monkeypatch))


class _CudaLike(torch.Tensor):
    is_cuda = True


def test_installed_wrapper_sends_cuda_tensors_to_the_kernel(monkeypatch):
    mu = _metrics_modules(monkeypatch)
    monkeypatch.setattr(SM, "compute_depth_metrics", lambda *a, **k: "kernel")
    monkeypatch.setattr(SM, "compute_depth_metrics_batched", lambda *a, **k: "kernel batched")
    try:
        S.install(metrics=True)
        x = torch.ones(2, 3)
        assert mu.compute_depth_metrics(x.as_subclass(_CudaLike), x) == "kernel"
        assert mu.compute_depth_metrics_batched(x.as_subclass(_CudaLike), x, x > 0) == "kernel batched"
        assert isinstance(mu.compute_depth_metrics(x, x), dict)
    finally:
        S.uninstall()


@pytest.mark.skipif(not reference_available(), reason="needs $SIMPLERECON_REF (the reference tree)")
def test_install_metrics_against_the_real_reference_module(monkeypatch):
    path = os.path.join(reference_root(), "utils", "metrics_utils.py")
    spec = importlib.util.spec_from_file_location("utils.metrics_utils", path)
    mu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mu)
    check_install(monkeypatch, _metrics_modules(monkeypatch, mu))
