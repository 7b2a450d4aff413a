"""CPU: the voxel down-sampling oracle (oracle/voxel_downsample_oracle.py, DESIGN §4.19) against a plain Python
restatement of the rule (a dict of voxels, float sums in input order), and the PyTorch op sequence the benchmark
times against the numpy oracle, bitwise."""
import math

import numpy as np
import pytest
import torch

from oracle import voxel_downsample_oracle as VD


def literal(points, s, colors=None):
    """The rule one point at a time: Python floats are IEEE fp64."""
    p = np.asarray(points, np.float32).astype(np.float64)
    b = [min(p[:, k]) - 0.5 * s for k in range(3)]
    vox = {}
    for i, q in enumerate(p):
        key = tuple(math.floor((float(q[k]) - b[k]) / s) for k in range(3))
        acc = vox.setdefault(key, [0.0] * 6 + [0])
        for k in range(3):
            acc[k] += float(q[k])
            if colors is not None:
                c = colors[i, k]
                acc[3 + k] += float(c) / 255.0 if colors.dtype == np.uint8 else float(c)
        acc[6] += 1
    keys = sorted(vox)
    pts = np.array([[vox[k][j] / vox[k][6] for j in range(3)] for k in keys]).astype(np.float32)
    cols = np.array([[vox[k][3 + j] / vox[k][6] for j in range(3)] for k in keys]).astype(np.float32)
    return pts, (cols if colors is not None else None), np.array([vox[k][6] for k in keys], np.int32)


@pytest.mark.parametrize("seed,s,n,spread", [(0, 0.02, 2000, 0.2), (1, 0.03, 1500, 0.05), (2, 0.02, 800, 5e-3),
                                             (3, 0.25, 1000, 2.0)])
def test_oracle_equals_literal_rule(seed, s, n, spread):
    rng = np.random.default_rng(seed)
    p = (rng.normal(size=(n, 3)) * spread - 3.0).astype(np.float32)
    for c in (None, rng.integers(0, 256, size=(n, 3)).astype(np.uint8), rng.random((n, 3))):
        got = VD.voxel_down_sample(p, s, c, long_run=4)       # both the rank loop and the accumulate path
        ref = literal(p, s, c)
        for g, r in zip(got, ref):
            if r is None:
                assert g is None
            else:
                np.testing.assert_array_equal(g.view(np.int32), r.view(np.int32))


def test_torch_op_sequence_equals_oracle():
    rng = np.random.default_rng(4)
    p = np.concatenate([rng.uniform(0, 0.3, size=(3000, 3)), 0.1 + rng.normal(scale=1e-3, size=(500, 3))])
    p = p.astype(np.float32)
    c = rng.integers(0, 256, size=(len(p), 3)).astype(np.uint8)
    ref = VD.voxel_down_sample(p, 0.02, c)
    got = VD.voxel_down_sample_torch(torch.from_numpy(p), 0.02, torch.from_numpy(c))
    for g, r in zip(got, ref):
        np.testing.assert_array_equal(g.numpy().view(np.int32), r.view(np.int32))


def test_extent_limit():
    VD.voxel_keys(np.array([[0, 0, 0], [2 ** 21 - 2, 0, 0]], np.float32), 1.0)
    with pytest.raises(ValueError):
        VD.voxel_keys(np.array([[0, 0, 0], [2 ** 21 - 1, 0, 0]], np.float32), 1.0)
