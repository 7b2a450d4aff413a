"""CPU: the restated kornia filters of oracle/normals_oracle.py on inputs with known answers — the blur's
impulse response is the tap vector (with the reflect fold at the border), Sobel of a linear ramp is 1
inside and 1/2 at the replicated border, a fronto-parallel plane has the normal (0, 0, 1) everywhere —
and the stand-ins compile under TorchScript, as the reference's scripted NormalGenerator needs."""
import torch

from oracle import normals_oracle as O
from simplerecon_b200.normals import gaussian_taps


def test_taps_match_the_expression_and_sum_to_one():
    for k, s in ((5, 2.0), (3, 1.0), (7, 3.0), (1, 2.0)):
        t = O.gaussian(k, s)
        assert t.dtype == torch.float32 and t.shape == (k,)
        assert torch.equal(t, gaussian_taps(k, s))
        assert abs(t.sum().item() - 1.0) < 1e-6 and torch.equal(t, t.flip(0))


def test_blur_impulse_response_is_the_tap_vector():
    k, s = 5, 2.0
    t = O.gaussian(k, s).double()
    x = torch.zeros(1, 1, 9, 11, dtype=torch.float64)
    x[0, 0, 4, 5] = 1.0                                    # interior impulse: the outer product of the taps
    out = O.gaussian_blur2d(x, (k, k), (s, s))
    assert torch.allclose(out[0, 0, 2:7, 3:8], torch.outer(t, t), atol=0, rtol=1e-15)
    assert abs(out.sum().item() - t.sum().item() ** 2) < 1e-12
    # impulse on the edge column: reflect does not repeat the edge pixel, so it is seen once per output
    x = torch.zeros(1, 1, 5, 8, dtype=torch.float64)
    x[:, :, :, 0] = 1.0
    out = O.gaussian_blur2d(x, (1, k), (s, s))[0, 0, 2]
    assert torch.allclose(out[:3], torch.stack([t[2], t[1], t[0]]), atol=0, rtol=1e-15)
    assert out[3:].abs().max().item() == 0.0
    # impulse one pixel inside: through the mirrored column -1 it is seen twice by columns 0 and 1
    x = torch.zeros(1, 1, 5, 8, dtype=torch.float64)
    x[:, :, :, 1] = 1.0
    out = O.gaussian_blur2d(x, (1, k), (s, s))[0, 0, 0]
    assert torch.allclose(out[:4], torch.stack([t[1] + t[3], t[2] + t[0], t[1], t[0]]), atol=0, rtol=1e-15)


def test_sobel_of_a_ramp():
    h, w = 6, 7
    v, u = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    g = O.spatial_gradient(torch.stack([u, v])[None])          # channel 0 ramps in x, channel 1 in y
    gx_of_x, gy_of_y = g[0, 0, 0], g[0, 1, 1]
    assert torch.all(gx_of_x[:, 1:-1] == 1.0) and torch.all(gx_of_x[:, [0, -1]] == 0.5)
    assert torch.all(gy_of_y[1:-1] == 1.0) and torch.all(gy_of_y[[0, -1]] == 0.5)
    assert torch.all(g[0, 0, 1] == 0.0) and torch.all(g[0, 1, 0] == 0.0)


def test_fronto_parallel_plane_faces_the_camera():
    # power-of-two focal lengths: the inverse and every ray are exact in fp32, so the fp32 result is
    # (0, 0, 1) to the last bit rather than to the rounding of a GEMM
    K = torch.eye(4)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = 128.0, 64.0, 16.5, 11.25
    invK = torch.inverse(K)[None].repeat(2, 1, 1)
    # (a depth of 2.5 in fp32 is 1.5e-6 off at the border rows: conv2d's rounding of the blurred depth)
    for dt, d in ((torch.float32, 2.0), (torch.float64, 2.0), (torch.float64, 2.5)):
        n = O.normal_generator(torch.full((2, 1, 24, 32), d, dtype=dt), invK.to(dt))
        assert torch.all((n[:, 0].abs() <= 1e-6) & (n[:, 1].abs() <= 1e-6) & ((n[:, 2] - 1).abs() <= 1e-6))


def test_non_finite_depth_spreads_over_the_full_window():
    depth = torch.full((1, 1, 15, 15), 2.0)
    depth[0, 0, 7, 7] = float("nan")
    invK = torch.inverse(torch.tensor([[100.0, 0, 7, 0], [0, 100.0, 7, 0], [0, 0, 1, 0], [0, 0, 0, 1]]))[None]
    bad = ~O.all_finite(O.normal_generator(depth, invK))[0]
    assert bad[4:11, 4:11].all() and bad.sum().item() == 49     # radius 2 (blur) + 1 (Sobel)


def test_stand_ins_compile_under_torchscript():
    blur = torch.jit.script(O.gaussian_blur2d)
    grad = torch.jit.script(O.spatial_gradient)
    x = torch.rand(2, 1, 9, 10)
    assert torch.equal(blur(x, (5, 5), (2.0, 2.0)), O.gaussian_blur2d(x, (5, 5), (2.0, 2.0)))
    assert torch.equal(grad(x), O.spatial_gradient(x))

    class UsesThem(torch.jit.ScriptModule):          # the shape of the reference's NormalGenerator.forward
        def __init__(self):
            super().__init__()
            self.kernel_size = 5
            self.std = 2.0

        @torch.jit.script_method
        def forward(self, d):
            return O.spatial_gradient(O.gaussian_blur2d(d, (self.kernel_size, self.kernel_size), (self.std, self.std)))

    assert UsesThem()(x).shape == (2, 1, 2, 9, 10)
