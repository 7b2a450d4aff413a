"""``b200cv::*`` — the fused sweeps registered as first-class torch operators.

SURVEY.md §8b asks, next to the C ABI, for a torch-library registration so the sweeps can
be called as ``torch.ops.b200cv.dot_forward(...)`` / ``mlp_forward(...)``: they then have a
schema, a fake (meta) kernel for shape propagation under ``FakeTensorMode`` /
``torch.compile`` / ``torch.export``, and an autograd formula, and they work under
``torch.inference_mode()``.  Only a CUDA kernel is registered for each: called with CPU
tensors they raise ``NotImplementedError`` from the dispatcher — there is no fallback.

Every CUDA kernel here is one call into ``libsrcv_b200.so`` (include/srcv_b200.h):

================================  ==========================================================
``b200cv::dot_forward``           ``srcv_dot_forward_f32``  — reference
                                  ``CostVolumeManager.build_cost_volume`` + argmax of
                                  ``forward`` (modules/cost_volume.py:237-335, :374-378)
``b200cv::dot_backward``          ``srcv_dot_backward_f32`` — autograd of :305-333 w.r.t.
                                  ``cur_feats`` / ``src_feats``
``b200cv::mlp_forward``           ``srcv_mlp_forward_f32``  — reference
                                  ``FeatureVolumeManager.build_cost_volume`` (:451-736) /
                                  ``FastFeatureVolumeManager.build_cost_volume`` (:967-1164)
``b200cv::mlp_backward``          ``srcv_mlp_backward_f32`` — autograd of the same composite
                                  w.r.t. the two feature inputs and the six MLP parameters
================================  ==========================================================

``planes`` is either ``(B, D)`` (one depth per plane, the reference's default log-spaced
planes of :100-136 after ``[:, :, 0, 0]``) or ``(B, D, H, W)`` (per-pixel planes, the
``depth_planes_bdhw`` argument of :247).  The manager classes in ``cost_volume.py`` are the
drop-in surface; these operators are the same sweeps without the module around them.
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import torch
from torch import Tensor

from . import _native

__all__ = ["dot_forward", "dot_backward", "mlp_forward", "mlp_backward"]


# ---------------------------------------------------------------------------------------------
# argument checks shared by the real and the fake kernels (so both raise on the same inputs)
# ---------------------------------------------------------------------------------------------
def _check_shapes(cur: Tensor, src: Tensor, E: Tensor, Ks: Tensor, invK: Tensor, planes: Tensor,
                  poses: Tensor | None = None) -> Tuple[int, int, int, int, int, int, bool]:
    if src.dim() != 5:
        raise ValueError("src_feats must be (B,K,C,H,W)")
    B, K, Cc, H, W = src.shape
    if tuple(cur.shape) != (B, Cc, H, W):
        raise ValueError(f"cur_feats shape {tuple(cur.shape)} != {(B, Cc, H, W)}")
    for name, t, shp in (("src_extrinsics", E, (B, K, 4, 4)), ("src_Ks", Ks, (B, K, 4, 4)),
                         ("cur_invK", invK, (B, 4, 4))):
        if tuple(t.shape) != shp:
            raise ValueError(f"{name} shape {tuple(t.shape)} != {shp}")
    if poses is not None and tuple(poses.shape) != (B, K, 4, 4):
        raise ValueError(f"src_poses shape {tuple(poses.shape)} != {(B, K, 4, 4)}")
    if planes.dim() == 2 and planes.shape[0] == B:
        per_pixel = False
    elif planes.dim() == 4 and tuple(planes.shape[::2]) == (B, H) and planes.shape[3] == W:
        per_pixel = True
    else:
        raise ValueError(f"planes must be (B,D) or (B,D,H,W); got {tuple(planes.shape)}")
    D = planes.shape[1]
    if D < 1:
        raise ValueError("planes holds no depth plane")
    for name, t in (("cur_feats", cur), ("src_feats", src), ("src_extrinsics", E), ("src_Ks", Ks),
                    ("cur_invK", invK), ("planes", planes)) + ((("src_poses", poses),) if poses is not None else ()):
        if t.dtype != torch.float32:
            raise ValueError(f"{name} must be float32 (got {t.dtype})")
    return B, K, Cc, H, W, D, per_pixel


def _c16(t: Tensor) -> Tensor:
    t = t.contiguous()
    return t.clone() if t.data_ptr() % 16 else t      # the kernels use 16-byte vector loads


def _ptr(t: Tensor | None):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _planes_struct(planes: Tensor, per_pixel: bool) -> _native.Planes:
    pl = _native.Planes()
    pl.mode = _native.PLANES_PER_PIXEL if per_pixel else _native.PLANES_PER_PLANE
    pl.planes = planes.data_ptr()
    pl.min_depth = pl.max_depth = pl.ramp = pl.planes_out = None
    return pl


def _marshal(cur_feats: Tensor, src_feats: Tensor, src_extrinsics: Tensor, src_Ks: Tensor, cur_invK: Tensor,
             planes: Tensor, src_poses: Tensor | None = None):
    """Checks the operator arguments (``_check_shapes``) and lays them out for the C ABI: returns
    ``(shape, cams, planes_struct, tensors)``, ``tensors`` being the dense, 16-byte aligned copies
    ``(cur, src, E, P, Ks, invK, planes)`` the structs point into (``P`` None without poses); they must
    stay alive until the call returns."""
    B, K, Cc, H, W, D, per_pixel = _check_shapes(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK,
                                                 planes, src_poses)
    cur, src, E, Ks, invK, pln = map(_c16, (cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes))
    P = _c16(src_poses) if src_poses is not None else None
    cams = _native.Cameras(E.data_ptr(), P.data_ptr() if P is not None else None, Ks.data_ptr(), invK.data_ptr())
    return _native.Shape(B, K, Cc, H, W, D), cams, _planes_struct(pln, per_pixel), (cur, src, E, P, Ks, invK, pln)


# ---------------------------------------------------------------------------------------------
# the forward launches of both the operators and the managers (their callers check the arguments)
# ---------------------------------------------------------------------------------------------
def _dot_sweep(shape: _native.Shape, cur: Tensor, src: Tensor, cams: _native.Cameras, pl: _native.Planes,
               want_lowest: bool) -> Tuple[Tensor, Tensor | None]:
    """``(cost (B,D,H,W), lowest_cost (B,H,W) or None)``: one ``srcv_dot_forward_f32`` call on the
    current stream of ``src``'s device."""
    lib = _native.load()
    dev = src.device
    with torch.cuda.device(dev):
        cost = torch.empty(shape.B, shape.D, shape.H, shape.W, device=dev, dtype=torch.float32)
        lowest = torch.empty(shape.B, shape.H, shape.W, device=dev, dtype=torch.float32) if want_lowest else None
        n = lib.srcv_dot_workspace_bytes(C.byref(shape))
        ws = torch.empty(n, device=dev, dtype=torch.uint8)
        _native.check(lib.srcv_dot_forward_f32(
            C.byref(shape), _ptr(cur), _ptr(src), C.byref(cams), C.byref(pl), _ptr(cost), _ptr(lowest),
            _ptr(ws), n, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return cost, lowest


def _mlp_sweep(shape: _native.Shape, cur: Tensor, src: Tensor, cams: _native.Cameras, pl: _native.Planes,
               w: _native.MlpWeights, want_lowest: bool, want_mask: bool
               ) -> Tuple[Tensor, Tensor | None, Tensor | None]:
    """``(cost (B,D,H,W), lowest_cost (B,H,W) or None, overall_mask (B,H,W) bool or None)``: one
    ``srcv_mlp_forward_f32`` call on the current stream of ``src``'s device.  Without
    ``w.packed_image`` the tensor-core kernel packs the weights into its workspace."""
    lib = _native.load()
    dev = src.device
    with torch.cuda.device(dev):
        cost = torch.empty(shape.B, shape.D, shape.H, shape.W, device=dev, dtype=torch.float32)
        lowest = torch.empty(shape.B, shape.H, shape.W, device=dev, dtype=torch.float32) if want_lowest else None
        mask = torch.empty(shape.B, shape.H, shape.W, device=dev, dtype=torch.uint8) if want_mask else None
        n = lib.srcv_mlp_workspace_bytes(C.byref(shape), C.byref(w))
        if n == 0:
            raise NotImplementedError(f"MLP widths ({w.hidden1},{w.hidden2}) are not supported by the fused kernels")
        ws = torch.empty(n, device=dev, dtype=torch.uint8)
        _native.check(lib.srcv_mlp_forward_f32(
            C.byref(shape), _ptr(cur), _ptr(src), C.byref(cams), C.byref(pl), C.byref(w), _ptr(cost),
            _ptr(lowest), _ptr(mask), _ptr(ws), n, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return cost, lowest, (mask.bool() if mask is not None else None)


# ---------------------------------------------------------------------------------------------
# b200cv::dot_forward / dot_backward
# ---------------------------------------------------------------------------------------------
def _dot_forward(cur_feats: Tensor, src_feats: Tensor, src_extrinsics: Tensor, src_Ks: Tensor,
                 cur_invK: Tensor, planes: Tensor) -> Tuple[Tensor, Tensor]:
    """``(cost (B,D,H,W), lowest_cost (B,H,W))`` of the dot-product sweep."""
    shape, cams, pl, (cur, src, *keep) = _marshal(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes)
    return _dot_sweep(shape, cur, src, cams, pl, want_lowest=True)


dot_forward = torch.library.custom_op("b200cv::dot_forward", _dot_forward, mutates_args=(), device_types="cuda")


@dot_forward.register_fake
def _(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes):
    B, K, Cc, H, W, D, _pp = _check_shapes(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes)
    return src_feats.new_empty((B, D, H, W)), src_feats.new_empty((B, H, W))


def _dot_backward(grad_cost: Tensor, cur_feats: Tensor, src_feats: Tensor, src_extrinsics: Tensor,
                  src_Ks: Tensor, cur_invK: Tensor, planes: Tensor) -> Tuple[Tensor, Tensor]:
    """``(dL/dcur_feats, dL/dsrc_feats)`` given ``dL/dcost``."""
    shape, cams, pl, (cur, src, *keep) = _marshal(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes)
    bdhw = (shape.B, shape.D, shape.H, shape.W)
    if tuple(grad_cost.shape) != bdhw or grad_cost.dtype != torch.float32:
        raise ValueError(f"grad_cost must be float32 {bdhw}")
    lib = _native.load()
    dev = src.device
    g = _c16(grad_cost)
    with torch.cuda.device(dev):
        gcur, gsrc = torch.empty_like(cur), torch.empty_like(src)
        n = lib.srcv_dot_backward_workspace_bytes(C.byref(shape))
        ws = torch.empty(n, device=dev, dtype=torch.uint8)
        _native.check(lib.srcv_dot_backward_f32(
            C.byref(shape), _ptr(cur), _ptr(src), C.byref(cams), C.byref(pl), _ptr(g), _ptr(gcur), _ptr(gsrc),
            _ptr(ws), n, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return gcur, gsrc


dot_backward = torch.library.custom_op("b200cv::dot_backward", _dot_backward, mutates_args=(), device_types="cuda")


@dot_backward.register_fake
def _(grad_cost, cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes):
    _check_shapes(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes)
    return torch.empty_like(cur_feats, memory_format=torch.contiguous_format), \
        torch.empty_like(src_feats, memory_format=torch.contiguous_format)


def _dot_setup_context(ctx, inputs, output):
    ctx.save_for_backward(*inputs)
    ctx.mark_non_differentiable(output[1])     # lowest_cost comes from an argmax


def _dot_autograd(ctx, grad_cost, _grad_lowest):
    cur, src, E, Ks, invK, planes = ctx.saved_tensors
    gcur = gsrc = None
    if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
        gcur, gsrc = dot_backward(grad_cost.contiguous(), cur, src, E, Ks, invK, planes)
    # cameras and plane depths get no gradient (the reference trains with fixed poses)
    return gcur, gsrc, None, None, None, None


dot_forward.register_autograd(_dot_autograd, setup_context=_dot_setup_context)


# ---------------------------------------------------------------------------------------------
# b200cv::mlp_forward
# ---------------------------------------------------------------------------------------------
def _check_mlp(K: int, Cc: int, w1, b1, w2, b2, w3, b3) -> Tuple[int, int]:
    F = Cc * (K + 1) + 10 * K + 4          # channel bookkeeping of modules/cost_volume.py:420-435
    if w1.dim() != 2 or w1.shape[1] != F:
        raise ValueError(f"w1 must be (H1,{F}) for K={K}, C={Cc}; got {tuple(w1.shape)}")
    h1 = w1.shape[0]
    if w2.dim() != 2 or w2.shape[1] != h1:
        raise ValueError(f"w2 must be (H2,{h1}); got {tuple(w2.shape)}")
    h2 = w2.shape[0]
    if tuple(w3.shape) != (1, h2) or tuple(b1.shape) != (h1,) or tuple(b2.shape) != (h2,) \
            or tuple(b3.shape) != (1,):
        raise ValueError("MLP parameter shapes must be w1 (H1,F), b1 (H1), w2 (H2,H1), b2 (H2), w3 (1,H2), b3 (1)")
    for t in (w1, b1, w2, b2, w3, b3):
        if t.dtype != torch.float32:
            raise ValueError("MLP parameters must be float32")
    return h1, h2


def _mlp_forward(cur_feats: Tensor, src_feats: Tensor, src_extrinsics: Tensor, src_poses: Tensor,
                 src_Ks: Tensor, cur_invK: Tensor, planes: Tensor, w1: Tensor, b1: Tensor, w2: Tensor,
                 b2: Tensor, w3: Tensor, b3: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """``(cost (B,D,H,W), lowest_cost (B,H,W), overall_mask (B,H,W) bool)`` of the metadata-MLP
    sweep; the MLP is ``F→H1→H2→1`` with LeakyReLU(0.01) (modules/networks.py:129-147)."""
    shape, cams, pl, (cur, src, *keep) = _marshal(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK,
                                                  planes, src_poses)
    h1, h2 = _check_mlp(shape.K, shape.C, w1, b1, w2, b2, w3, b3)
    ws_t = [_c16(t.detach()) for t in (w1, b1, w2, b2, w3, b3)]
    w = _native.MlpWeights(*[t.data_ptr() for t in ws_t], h1, h2)
    return _mlp_sweep(shape, cur, src, cams, pl, w, want_lowest=True, want_mask=True)


mlp_forward = torch.library.custom_op("b200cv::mlp_forward", _mlp_forward, mutates_args=(), device_types="cuda")


@mlp_forward.register_fake
def _(cur_feats, src_feats, src_extrinsics, src_poses, src_Ks, cur_invK, planes, w1, b1, w2, b2, w3, b3):
    B, K, Cc, H, W, D, _pp = _check_shapes(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes,
                                           src_poses)
    _check_mlp(K, Cc, w1, b1, w2, b2, w3, b3)
    return (src_feats.new_empty((B, D, H, W)), src_feats.new_empty((B, H, W)),
            src_feats.new_empty((B, H, W), dtype=torch.bool))


def _mlp_backward(grad_cost: Tensor, cur_feats: Tensor, src_feats: Tensor, src_extrinsics: Tensor,
                  src_poses: Tensor, src_Ks: Tensor, cur_invK: Tensor, planes: Tensor, w1: Tensor, b1: Tensor,
                  w2: Tensor, b2: Tensor, w3: Tensor, b3: Tensor
                  ) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """``(dL/dcur_feats, dL/dsrc_feats, dL/dw1, dL/db1, dL/dw2, dL/db2, dL/dw3, dL/db3)`` given
    ``dL/dcost`` — a recompute kernel: nothing of the forward is needed but its inputs."""
    shape, cams, pl, (cur, src, *keep) = _marshal(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK,
                                                  planes, src_poses)
    h1, h2 = _check_mlp(shape.K, shape.C, w1, b1, w2, b2, w3, b3)
    bdhw = (shape.B, shape.D, shape.H, shape.W)
    if tuple(grad_cost.shape) != bdhw or grad_cost.dtype != torch.float32:
        raise ValueError(f"grad_cost must be float32 {bdhw}")
    lib = _native.load()
    dev = src.device
    g = _c16(grad_cost)
    ws_t = [_c16(t.detach()) for t in (w1, b1, w2, b2, w3, b3)]
    w = _native.MlpWeights(*[t.data_ptr() for t in ws_t], h1, h2)
    with torch.cuda.device(dev):
        gcur, gsrc = torch.empty_like(cur), torch.empty_like(src)
        gw = [torch.empty_like(t) for t in ws_t]
        grads = _native.MlpGrads(*[t.data_ptr() for t in gw])
        n = lib.srcv_mlp_backward_workspace_bytes(C.byref(shape), C.byref(w))
        if n == 0:
            raise NotImplementedError("metadata-MLP backward: at most 208 input features, hidden widths <= 128")
        ws = torch.empty(n, device=dev, dtype=torch.uint8)
        _native.check(lib.srcv_mlp_backward_f32(
            C.byref(shape), _ptr(cur), _ptr(src), C.byref(cams), C.byref(pl), C.byref(w), _ptr(g), _ptr(gcur),
            _ptr(gsrc), C.byref(grads), _ptr(ws), n, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return (gcur, gsrc, *gw)


mlp_backward = torch.library.custom_op("b200cv::mlp_backward", _mlp_backward, mutates_args=(), device_types="cuda")


@mlp_backward.register_fake
def _(grad_cost, cur_feats, src_feats, src_extrinsics, src_poses, src_Ks, cur_invK, planes, w1, b1, w2, b2, w3, b3):
    B, K, Cc, H, W, D, _pp = _check_shapes(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK, planes,
                                           src_poses)
    _check_mlp(K, Cc, w1, b1, w2, b2, w3, b3)
    c = torch.contiguous_format
    return tuple(torch.empty_like(t, memory_format=c) for t in (cur_feats, src_feats, w1, b1, w2, b2, w3, b3))


def _mlp_setup_context(ctx, inputs, output):
    ctx.save_for_backward(*inputs)
    ctx.mark_non_differentiable(output[1], output[2])      # lowest_cost (argmax), overall mask (bool)


def _mlp_autograd(ctx, grad_cost, _grad_lowest, _grad_mask):
    cur, src, E, P, Ks, invK, planes, w1, b1, w2, b2, w3, b3 = ctx.saved_tensors
    need = ctx.needs_input_grad
    g = [None] * 13
    if any(need[i] for i in (0, 1, 7, 8, 9, 10, 11, 12)):
        out = mlp_backward(grad_cost.contiguous(), cur, src, E, P, Ks, invK, planes, w1, b1, w2, b2, w3, b3)
        g[0], g[1] = out[0], out[1]
        g[7:13] = out[2:8]
    return tuple(g)


mlp_forward.register_autograd(_mlp_autograd, setup_context=_mlp_setup_context)
