"""CPU oracle for SimpleRecon's plane-sweep cost-volume path.

TEST INFRASTRUCTURE — NOT PRODUCT CODE.  Only ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import this file.
The shipped package (``simplerecon_b200``) never does; it fails loudly when its CUDA
library is missing instead of falling back to anything in here.

Parity pin: the reference holds no tests or golden vectors for this path
(SURVEY.md §8c), so this restatement is pinned against the *reference's own classes*
(imported unmodified by ``oracle/ref_import.py``) through their stored outputs —
``tests/test_oracle_vs_reference.py`` (``tests/golden/reference/``) and the committed fixtures
``tests/golden/*.npz`` made by ``tests/golden/make_golden.py``.

What is restated (all citations relative to the reference tree):

* depth planes                    modules/cost_volume.py:100-136 (ramp built at :68-70)
* back-projection                 utils/geometry_utils.py:34-48 (+0.5 pixel centres), :51-59
* projection + guarded divide     utils/geometry_utils.py:72-89 (eps=1e-8, :66-69)
* grid normalisation              modules/cost_volume.py:199, :587 (uv_scale built :290-295)
* bilinear / zeros / align_corners=False sampling   F.grid_sample call at :201-212, :590-601
* depth-validity mask             modules/cost_volume.py:231-232, :622-623
* dot-product matching            modules/cost_volume.py:322-333
* argmax -> depth ("lowest_cost") modules/cost_volume.py:338-342, :374-378
* pose_distance                   utils/geometry_utils.py:178-191
* rays / ray angle                modules/cost_volume.py:641-688, utils/geometry_utils.py:168-173
* metadata concat order           modules/cost_volume.py:698-723
* MLP                             modules/networks.py:129-147 (LeakyReLU slope 0.01)
* overall mask (last plane wins)  modules/cost_volume.py:625-637, bounds test :90-95

Two samplers are provided.  ``sampler="explicit"`` spells the bilinear gather out
(the arithmetic the CUDA kernels implement, ATen-CUDA operation order);
``sampler="aten"`` calls ``F.grid_sample`` like the reference does, which makes the
oracle agree with the CPU reference to the last bit or two and is what the
``cpu_baseline`` leg times (it is the reference's op sequence: one Python iteration
per depth plane, ``grid_sample`` + ``normalize`` + ``cat`` + three ``Linear``s).
Works in fp32 and, for error budgeting, fp64 (pass double tensors).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

EPS_PROJ = 1e-8       # utils/geometry_utils.py:66
EPS_NORM = 1e-12      # F.normalize default
EPS_COS = 1e-5        # modules/cost_volume.py:687
LRELU_SLOPE = 0.01    # nn.LeakyReLU() default, modules/networks.py:140


# --------------------------------------------------------------------------- #
# geometry                                                                    #
# --------------------------------------------------------------------------- #
def depth_planes(min_depth, max_depth, num_depth_bins: int, dtype=torch.float32, device=None):
    """(D,) log-spaced plane depths — or (B,D) when the range holds one value per frame, which
    the reference's expression broadcasts ((B,1,1,1) against the (1,D,1,1) ramp).
    modules/cost_volume.py:68-70, :124-127."""
    min_depth = torch.as_tensor(min_depth, dtype=dtype, device=device).reshape(-1)
    max_depth = torch.as_tensor(max_depth, dtype=dtype, device=device).reshape(-1)
    # the reference builds the ramp in fp32 (register_buffer) and then .double()
    # converts the buffer, so an fp64 run still sees the fp32-rounded ramp.
    ramp = torch.linspace(0, 1, num_depth_bins).to(dtype).to(min_depth.device)
    out = torch.exp(torch.log(min_depth)[:, None] + torch.log(max_depth / min_depth)[:, None] * ramp[None])
    return out[0] if out.shape[0] == 1 else out


def pixel_centres(H: int, W: int, dtype=torch.float32, device=None):
    """(3, H*W) homogeneous pixel centres, xy order.  utils/geometry_utils.py:34-44."""
    v, u = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    return torch.stack(
        [u.reshape(-1) + 0.5, v.reshape(-1) + 0.5, torch.ones(H * W)], 0
    ).to(dtype).to(device)


def backproject_rays(cur_invK, H: int, W: int):
    """(B,3,N): r = invK[:3,:3] @ p.  utils/geometry_utils.py:56."""
    return torch.matmul(cur_invK[:, :3, :3], pixel_centres(H, W, cur_invK.dtype, cur_invK.device)[None])


def project(points_b3n, src_Ks, src_extrinsics):
    """Projects (B,3,N) points into every source view.

    Returns px, py, zprime each (B,K,N).  utils/geometry_utils.py:78-89.
    """
    B, K = src_Ks.shape[:2]
    P = torch.matmul(src_Ks, src_extrinsics)                      # (B,K,4,4)  :78
    ones = torch.ones_like(points_b3n[:, :1])
    X4 = torch.cat([points_b3n, ones], 1)                          # (B,4,N)    :57-58
    cam = torch.matmul(P[:, :, :3, :], X4[:, None])                # (B,K,3,N)  :80
    z = cam[:, :, 2]
    zp = z + EPS_PROJ                                              # :84
    scale = torch.where(z.abs() > EPS_PROJ, 1.0 / zp, torch.ones_like(zp))  # :83-85
    return cam[:, :, 0] * scale, cam[:, :, 1] * scale, zp


def sample_bilinear_zeros(src_bkchw, px, py, sampler: str = "explicit"):
    """Samples (B,K,C,H,W) features at pixel coords px,py (B,K,N) -> (B,K,C,N).

    bilinear, zeros padding, align_corners=False, coordinates normalised the way
    the reference does it (modules/cost_volume.py:199): g = 2*p*(1/size) - 1.
    """
    B, K, C, H, W = src_bkchw.shape
    N = px.shape[-1]
    dt = src_bkchw.dtype
    inv_w = torch.tensor(1.0 / W, dtype=dt)   # fp32 reciprocal as at :290-295
    inv_h = torch.tensor(1.0 / H, dtype=dt)
    gx = 2 * px * inv_w - 1
    gy = 2 * py * inv_h - 1
    if sampler == "aten":
        grid = torch.stack([gx, gy], -1).reshape(B * K, 1, N, 2)
        out = F.grid_sample(src_bkchw.reshape(B * K, C, H, W), grid, mode="bilinear",
                            padding_mode="zeros", align_corners=False)
        return out.reshape(B, K, C, N)
    # explicit restatement (ATen CUDA order: ((g+1)*size-1)/2)
    ix = ((gx + 1) * W - 1) / 2
    iy = ((gy + 1) * H - 1) / 2
    x0 = torch.floor(ix)
    y0 = torch.floor(iy)
    x1 = x0 + 1
    y1 = y0 + 1
    w_nw = (x1 - ix) * (y1 - iy)
    w_ne = (ix - x0) * (y1 - iy)
    w_sw = (x1 - ix) * (iy - y0)
    w_se = (ix - x0) * (iy - y0)
    flat = src_bkchw.reshape(B, K, C, H * W)

    def tap(xf, yf, w):
        ok = (xf >= 0) & (xf <= W - 1) & (yf >= 0) & (yf <= H - 1)
        # NaN / huge coordinates fail `ok`; clamp before the integer cast
        xi = torch.nan_to_num(xf, nan=0.0).clamp(0, W - 1).long()
        yi = torch.nan_to_num(yf, nan=0.0).clamp(0, H - 1).long()
        idx = (yi * W + xi)[:, :, None, :].expand(B, K, C, N)
        val = torch.gather(flat, 3, idx)
        wz = torch.where(ok, w, torch.zeros_like(w))
        return val * wz[:, :, None, :]

    return tap(x0, y0, w_nw) + tap(x1, y0, w_ne) + tap(x0, y1, w_sw) + tap(x1, y1, w_se)


def pose_distance(pose_bk44):
    """(comb, R_meas, t_meas) each (B,K).  utils/geometry_utils.py:178-191."""
    R = pose_bk44[..., :3, :3]
    t = pose_bk44[..., :3, 3]
    tr = R.diagonal(dim1=-2, dim2=-1).sum(-1)
    r_meas = torch.sqrt(2 * (1 - torch.minimum(torch.full_like(tr, 3.0), tr) / 3))
    t_meas = torch.linalg.vector_norm(t, dim=-1)
    comb = torch.sqrt(t_meas ** 2 + r_meas ** 2)
    return comb, r_meas, t_meas


def bounds_mask(px, py, H: int, W: int):
    """modules/cost_volume.py:90-95."""
    return (px > 2) & (px < W - 2) & (py > 2) & (py < H - 2)


def _planes_bdn(depth_planes_bdhw, min_depth, max_depth, B, D, H, W, dtype, device=None):
    """Returns (planes (B,D,N) view-able tensor, depth_planes_bdhw to hand back)."""
    if depth_planes_bdhw is None:
        d = depth_planes(min_depth, max_depth, D, dtype, device)
        depth_planes_bdhw = d.view(-1, D, 1, 1).expand(B, D, H, W)  # :129-134
    return depth_planes_bdhw.reshape(B, D, H * W), depth_planes_bdhw


# --------------------------------------------------------------------------- #
# dot-product volume (CostVolumeManager)                                      #
# --------------------------------------------------------------------------- #
def dot_volume(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK,
               min_depth=None, max_depth=None, num_depth_bins=64,
               depth_planes_bdhw=None, sampler="explicit"):
    """cost (B,D,H,W), depth_planes_bdhw.  modules/cost_volume.py:237-335."""
    B, K, C, H, W = src_feats.shape
    D = num_depth_bins if depth_planes_bdhw is None else depth_planes_bdhw.shape[1]
    planes, depth_planes_bdhw = _planes_bdn(depth_planes_bdhw, min_depth, max_depth,
                                            B, D, H, W, cur_feats.dtype, cur_feats.device)
    rays = backproject_rays(cur_invK, H, W)                        # (B,3,N)
    cur = cur_feats.reshape(B, 1, C, H * W)
    out = []
    for d in range(D):                                             # :305
        X = planes[:, d:d + 1] * rays                              # :57
        px, py, zp = project(X, src_Ks, src_extrinsics)
        warped = sample_bilinear_zeros(src_feats, px, py, sampler)  # (B,K,C,N)
        mask = (zp > 0).to(warped.dtype)                           # :231-232
        dot_k = (warped * cur).sum(2) * mask                       # :322-326
        out.append(dot_k.sum(1, keepdim=True))                     # :329
    return torch.cat(out, 1).reshape(B, D, H, W), depth_planes_bdhw


# --------------------------------------------------------------------------- #
# metadata-MLP volume (FeatureVolumeManager / FastFeatureVolumeManager)       #
# --------------------------------------------------------------------------- #
def mlp_apply(feat, weights):
    """feat (...,F) -> (...,).  modules/networks.py:134-147 (final activation stripped)."""
    W1, b1, W2, b2, W3, b3 = weights
    h = F.leaky_relu(F.linear(feat, W1, b1), LRELU_SLOPE)
    h = F.leaky_relu(F.linear(h, W2, b2), LRELU_SLOPE)
    return F.linear(h, W3, b3).squeeze(-1)


def feature_rows(cur_feats, src_feats, src_extrinsics, src_poses, src_Ks, cur_invK,
                 plane_b1n, sampler="explicit"):
    """The (B, N, F) MLP input of ONE depth plane, channel order of
    modules/cost_volume.py:698-723, plus px,py,zp for the mask."""
    B, K, C, H, W = src_feats.shape
    N = H * W
    rays = backproject_rays(cur_invK, H, W)
    X = plane_b1n * rays                                           # (B,3,N)
    px, py, zp = project(X, src_Ks, src_extrinsics)                # (B,K,N)
    warped = sample_bilinear_zeros(src_feats, px, py, sampler)     # (B,K,C,N)
    mask = (zp > 0).to(warped.dtype)
    cur = cur_feats.reshape(B, C, N)
    dot_k = (warped * cur[:, None]).sum(2) * mask                  # :691-695
    n_cur = F.normalize(X, dim=1, eps=EPS_NORM)                    # :641-648
    t = src_poses[:, :, :3, 3]                                     # (B,K,3)
    n_src = F.normalize(X[:, None] - t[..., None], dim=2, eps=EPS_NORM)  # geometry_utils.py:168-173
    ang = F.cosine_similarity(n_cur[:, None].expand_as(n_src), n_src, dim=2, eps=EPS_COS)  # :683-688
    comb, r_meas, t_meas = pose_distance(src_poses)
    ex = lambda s: s[:, :, None].expand(B, K, N)
    feat = torch.cat([
        warped.reshape(B, K * C, N),       # 0 .. K*C
        cur,                               # cur feats
        mask, zp,                          # m_k, z'_k
        plane_b1n.expand(B, 1, N),         # depth plane value
        dot_k, ang,
        n_cur, n_src.reshape(B, 3 * K, N),
        ex(comb), ex(r_meas), ex(t_meas),
    ], 1)                                                           # (B,F,N)
    return feat.permute(0, 2, 1), px, py, zp


def feature_volume(cur_feats, src_feats, src_extrinsics, src_poses, src_Ks, cur_invK,
                   weights, min_depth=None, max_depth=None, num_depth_bins=64,
                   depth_planes_bdhw=None, return_mask=False, sampler="explicit"):
    """cost (B,D,H,W), depth_planes_bdhw, overall_mask (B,H,W) bool or None.
    modules/cost_volume.py:451-736."""
    B, K, C, H, W = src_feats.shape
    D = num_depth_bins if depth_planes_bdhw is None else depth_planes_bdhw.shape[1]
    planes, depth_planes_bdhw = _planes_bdn(depth_planes_bdhw, min_depth, max_depth,
                                            B, D, H, W, cur_feats.dtype, cur_feats.device)
    out, overall = [], None
    for d in range(D):                                             # :557
        feat, px, py, zp = feature_rows(cur_feats, src_feats, src_extrinsics, src_poses,
                                        src_Ks, cur_invK, planes[:, d:d + 1], sampler)
        if return_mask:                                            # :625-637 (overwritten each plane)
            overall = (zp > 0).any(1) & bounds_mask(px, py, H, W).any(1)
        out.append(mlp_apply(feat, weights)[:, None])              # (B,1,N)
    cost = torch.cat(out, 1).reshape(B, D, H, W)
    if overall is not None:
        overall = overall.reshape(B, H, W)
    return cost, depth_planes_bdhw, overall


def lowest_cost(cost_bdhw, depth_planes_bdhw):
    """argmax over planes -> plane depth.  modules/cost_volume.py:338-342, :374-378."""
    idx = torch.argmax(cost_bdhw, 1, keepdim=True)
    return torch.gather(depth_planes_bdhw.expand_as(cost_bdhw), 1, idx).squeeze(1)


def forward_dot(cur_feats, src_feats, src_extrinsics, src_poses, src_Ks, cur_invK,
                min_depth, max_depth, num_depth_bins=64, depth_planes_bdhw=None,
                return_mask=False, sampler="explicit"):
    """Mirror of CostVolumeManager.forward (modules/cost_volume.py:345-380)."""
    cost, planes = dot_volume(cur_feats, src_feats, src_extrinsics, src_Ks, cur_invK,
                              min_depth, max_depth, num_depth_bins, depth_planes_bdhw, sampler)
    return cost, lowest_cost(cost, planes), planes, None


def forward_mlp(cur_feats, src_feats, src_extrinsics, src_poses, src_Ks, cur_invK,
                min_depth, max_depth, weights, num_depth_bins=64, depth_planes_bdhw=None,
                return_mask=False, sampler="explicit"):
    """Mirror of FeatureVolumeManager.forward."""
    cost, planes, mask = feature_volume(cur_feats, src_feats, src_extrinsics, src_poses,
                                        src_Ks, cur_invK, weights, min_depth, max_depth,
                                        num_depth_bins, depth_planes_bdhw, return_mask, sampler)
    return cost, lowest_cost(cost, planes), planes, mask


def mlp_weights_from_state_dict(sd, prefix="mlp.net."):
    return tuple(sd[f"{prefix}{i}.{n}"] for i in (0, 2, 4) for n in ("weight", "bias"))
