"""CPU: each kernel family's size query and its calls apply one size rule (host emulation, tests/emu).

One row per family: at a size on the limit the query is positive; one step past it the query returns 0 and a call
given a real workspace is refused, with SRCV_ERR_SHAPE (the mvloss view count: SRCV_ERR_UNSUPPORTED, a limit of the
build rather than a malformed shape), before anything is launched.  Sizes on the limit are only queried, never run."""
import ctypes as C

import pytest
import torch

from simplerecon_b200 import _native as N
from tests import emu

ERR_SHAPE, ERR_UNSUPPORTED = 2, 4
MVLOSS_MAX_VIEWS = 16      # include/srcv_b200.h: K <= 16
POINTS_MAX = 1 << 28       # mesh evaluation and voxel down-sampling
WS_BYTES = 1 << 20


@pytest.fixture(scope="module")
def lib():
    return emu.load_or_skip()


@pytest.fixture(scope="module")
def buf():
    """One 256-byte aligned host buffer: every pointer argument and the workspace (a refused call reads none)."""
    raw = torch.zeros(WS_BYTES + 256, dtype=torch.uint8)
    off = (-raw.data_ptr()) % 256
    return raw, raw.data_ptr() + off


def _frames(p, W):
    return N.TsdfFrames(p, p, p, None, 1, 1, W, 0.5, 5.0)


def _sparse(p, max_blocks=1):
    return N.SparseTsdf(p, max_blocks, 0, (C.c_float * 3)(), 0.1, 3.0, 100.0)


def _tsdf(lib, p, W):
    f = _frames(p, W)
    v = N.TsdfVolume(p, p, 8, 8, 8, (C.c_float * 3)(), 0.1, 3.0, 100.0)
    return (lib.srcv_tsdf_workspace_bytes(C.byref(f)),
            lambda: lib.srcv_tsdf_integrate_f16(C.byref(v), C.byref(f), p, WS_BYTES, None))


def _sparse_frames(lib, p, W):
    f, v = _frames(p, W), _sparse(p)
    return (lib.srcv_sparse_tsdf_workspace_bytes(C.byref(f)),
            lambda: lib.srcv_sparse_tsdf_integrate_f16(C.byref(v), C.byref(f), p, WS_BYTES, None))


def _sparse_state(lib, p, max_blocks):
    v = _sparse(p, max_blocks)
    return lib.srcv_sparse_tsdf_state_bytes(C.byref(v)), lambda: lib.srcv_sparse_tsdf_reset(C.byref(v), None)


def _sparse_mesh(lib, p, blocks):
    v, a = _sparse(p, 4), N.SparseMeshArgs(blocks, (C.c_float * 3)(), 0, 0)
    return (lib.srcv_sparse_tsdf_mesh_workspace_bytes(C.byref(a)),
            lambda: lib.srcv_sparse_tsdf_mesh_count(C.byref(v), C.byref(a), p, p, WS_BYTES, None))


def _mesh(lib, p, X):
    a = N.MeshArgs(p, p, X, 2, 2, (C.c_float * 3)(), 0.1, 0, 0)
    return lib.srcv_mesh_workspace_bytes(C.byref(a)), lambda: lib.srcv_mesh_count(C.byref(a), p, p, WS_BYTES, None)


def _mvs(lib, p, H):
    s = N.MvsScan(p, p, p, p, p, 2, H, 8)
    return (lib.srcv_mvs_workspace_bytes(C.byref(s)),
            lambda: lib.srcv_mvs_consistency_f32(C.byref(s), 0, 0.01, 1, p, p, p, p, WS_BYTES, 0, None))


def _mvloss(lib, p, B, K):
    a = N.MvLossArgs(p, p, p, p, p, p, p, B, K, 1, 1)
    return (lib.srcv_mvloss_workspace_bytes(C.byref(a)),
            lambda: lib.srcv_mvloss_forward_f32(C.byref(a), p, None, None, p, WS_BYTES, None))


def _voxel_ds(lib, p, n):
    return (lib.srcv_voxel_down_sample_workspace_bytes(n),
            lambda: lib.srcv_voxel_down_sample_f32(p, n, 0.1, None, 0, p, None, p, p, p, p, WS_BYTES, None))


def _si_loss(lib, p, n):
    return (lib.srcv_si_loss_workspace_bytes(n),
            lambda: lib.srcv_si_loss_forward_f32(p, p, n, 0.85, p, p, WS_BYTES, None))


# (family, make(lib, ptr, size) -> (query result, call), size on the limit, size just past it, refusal status)
ROWS = [
    ("tsdf_frames_W", _tsdf, 2048, 2049, ERR_SHAPE),
    ("sparse_frames_W", _sparse_frames, 2048, 2049, ERR_SHAPE),
    ("sparse_max_blocks", _sparse_state, 1 << 26, (1 << 26) + 1, ERR_SHAPE),
    ("sparse_mesh_blocks", _sparse_mesh, 0, -1, ERR_SHAPE),
    ("mesh_X", _mesh, 65535, 65536, ERR_SHAPE),
    ("mvs_H", _mvs, 2, 1, ERR_SHAPE),
    ("mvloss_B", lambda lib, p, B: _mvloss(lib, p, B, 1), 65535, 65536, ERR_SHAPE),
    ("mvloss_K", lambda lib, p, K: _mvloss(lib, p, 1, K), MVLOSS_MAX_VIEWS, MVLOSS_MAX_VIEWS + 1, ERR_UNSUPPORTED),
    ("voxel_ds_points", _voxel_ds, POINTS_MAX, POINTS_MAX + 1, ERR_SHAPE),
    ("si_loss_n", _si_loss, (1 << 31) - 1, 1 << 31, ERR_SHAPE),
]


@pytest.mark.parametrize("family,make,at,past,status", ROWS, ids=[r[0] for r in ROWS])
def test_query_and_call_share_the_limit(lib, buf, family, make, at, past, status):
    p = C.c_void_p(buf[1])
    n_at, _ = make(lib, p, at)
    assert n_at > 0, f"{family}: the size query refuses {at}, which its calls accept"
    n_past, call = make(lib, p, past)
    assert n_past == 0, f"{family}: the size query sizes {past} ({n_past} bytes), which its calls refuse"
    n0 = lib.srcv_launch_count()
    assert call() == status, lib.srcv_last_error().decode()
    assert lib.srcv_launch_count() == n0
