"""K10: the wgmma 3xTF32 product (csrc/gemm.cu, b2rl_gemm_tf32x3) against an fp64 product.

Tolerance: on these random-sign operands every element within 2^-18 * (|A| . |B|^T) of the
fp64 result.  This is what random signs give, not a worst case: the tensor core truncates on
every accumulation, so on same-sign data the error grows with the number of k steps per split
(2^-14 at K = 8192 in one split).  tests/test_tensor_core_fp64_gpu.py derives the K-dependent
bound that holds for any data and checks every path against it.  The error also sits next to
cuBLAS' own fp32 SGEMM error, which the test prints and bounds too (<= 4x cuBLAS' max error
+ 1e-6).  The shapes are the Rainbow / DQN
layers at B = 512 (pfrl/q_functions/dueling_dqn.py:67-129) in all three orientations (forward,
dX, dW), ragged edges, unaligned leading dimensions, strided (chunked) inputs.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref64(a, b, a_mn, b_mn):
    a64 = a.double().t() if a_mn else a.double()
    b64 = b.double().t() if b_mn else b.double()
    return a64 @ b64.t(), a64.abs() @ b64.abs().t()


def _f32(a, b, a_mn, b_mn):
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        af = a.t() if a_mn else a
        bf = b.t() if b_mn else b
        return af @ bf.t()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


CASES = [
    # M, N, K, a_mn, b_mn
    (512, 1024, 3136, False, False),   # main_stream forward
    (512, 3136, 1024, False, True),    # main_stream dX
    (1024, 3136, 512, True, True),     # main_stream dW
    (512, 918, 512, False, False),     # a_stream forward (18 actions x 51 atoms)
    (512, 512, 918, False, True),      # a_stream dX (lda = 918: unaligned rows)
    (918, 512, 512, True, True),       # a_stream dW
    (512, 51, 512, False, False),      # v_stream forward
    (51, 512, 512, True, True),        # v_stream dW
    (32, 512, 3136, False, False),     # DQN head at B = 32
    (130, 70, 45, False, False),       # ragged everything, K tail
    (130, 70, 45, True, False),
    (130, 70, 45, False, True),
    (5, 7, 9, True, True),
    (128, 128, 32, False, False),      # exactly one tile, one k block
    (256, 256, 8192, False, False),    # deep K: many splits
]


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", CASES)
def test_gemm_vs_fp64(M, N, K, a_mn, b_mn):
    from pfrl_b200.ops.linear import gemm

    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g)
    b = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    # a spread of magnitudes, exact zeros and denormal-sized values
    a[::3] *= 37.5
    b[::5] *= 1e-3
    a[0, :] = 0
    c = gemm(a, b, a_mn_major=a_mn, b_mn_major=b_mn)
    torch.cuda.synchronize()
    ref, bound = _ref64(a, b, a_mn, b_mn)
    err = (c.double() - ref).abs()
    err_cublas = (_f32(a, b, a_mn, b_mn).double() - ref).abs()
    worst = float((err / (bound + 1e-300)).max())
    print(f"[gemm {M}x{N}x{K} a_mn={a_mn} b_mn={b_mn}] max err {float(err.max()):.3e} "
          f"(cuBLAS fp32 {float(err_cublas.max()):.3e}), rel-to-bound {worst:.3e}")
    assert c.shape == (M, N)
    assert torch.isfinite(c).all()
    assert worst <= 2.0 ** -18
    assert float(err.max()) <= 4 * float(err_cublas.max()) + 1e-6


def test_gemm_bias_relu_and_determinism():
    from pfrl_b200.ops.linear import gemm

    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(300, 3136, device="cuda", generator=g)
    b = torch.randn(200, 3136, device="cuda", generator=g)
    bias = torch.randn(200, device="cuda", generator=g)
    c1 = gemm(a, b, bias=bias, relu=True)
    c2 = gemm(a, b, bias=bias, relu=True)
    ref = torch.relu(a.double() @ b.double().t() + bias.double())
    assert torch.equal(c1, c2)  # split-K partials are summed in a fixed order
    assert (c1.double() - ref).abs().max() < 1e-3
    assert (c1 >= 0).all()


def test_gemm_strided_operands_read_in_place():
    from pfrl_b200.ops.linear import gemm

    g = torch.Generator(device="cuda").manual_seed(6)
    h = torch.randn(512, 1024, device="cuda", generator=g)
    w = torch.randn(918, 512, device="cuda", generator=g)
    h_a, h_v = torch.chunk(h, 2, dim=1)  # row stride 1024, second half starts at column 512
    for part in (h_a, h_v):
        c = gemm(part, w)
        ref = part.double() @ w.double().t()
        assert (c.double() - ref).abs().max() < 2e-4


def test_linear_autograd_matches_fp64():
    from pfrl_b200.ops.linear import linear

    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(512, 3136, device="cuda", generator=g, requires_grad=True)
    w = (torch.randn(1024, 3136, device="cuda", generator=g) * 0.02).requires_grad_()
    b = torch.randn(1024, device="cuda", generator=g, requires_grad=True)
    gy = torch.randn(512, 1024, device="cuda", generator=g)
    y = linear(x, w, b)
    gx, gw, gb = torch.autograd.grad(y, (x, w, b), gy)
    x64, w64, b64 = (t.detach().double().requires_grad_() for t in (x, w, b))
    y64 = torch.nn.functional.linear(x64, w64, b64)
    gx64, gw64, gb64 = torch.autograd.grad(y64, (x64, w64, b64), gy.double())
    for name, got, want in (("y", y, y64), ("gx", gx, gx64), ("gw", gw, gw64), ("gb", gb, gb64)):
        rel = float((got.double() - want).abs().max() / want.abs().max())
        print(f"[linear] {name}: rel err {rel:.3e}")
        assert rel < 5e-6, name


def test_rainbow_head_uses_the_tensor_core_path(monkeypatch):
    """The Rainbow network's dense layers go through b2rl_gemm_tf32x3 on CUDA and agree with the
    cuBLAS path (B2RL_LINEAR=cublas) to fp32 round-off."""
    from pfrl_b200.nn.noisy_chain import to_factorized_noisy
    from pfrl_b200.ops import linear as lin
    from pfrl_b200.q_functions import DistributionalDuelingDQN

    torch.manual_seed(0)
    q = DistributionalDuelingDQN(18, 51, -10, 10).cuda()
    x = torch.rand(512, 4, 84, 84, device="cuda")
    calls = []
    real = lin.gemm
    monkeypatch.setattr(lin, "gemm", lambda *a, **k: (calls.append(1), real(*a, **k))[1])
    q(x)
    assert len(calls) == 2  # default policy (ops.linear.worth_it): main_stream and a_stream
    calls.clear()
    monkeypatch.setenv("B2RL_LINEAR", "tcgen05")
    out_tc = q(x).q_values
    assert len(calls) == 3  # main_stream, a_stream, v_stream
    monkeypatch.setenv("B2RL_LINEAR", "cublas")
    out_cb = q(x).q_values
    assert (out_tc - out_cb).abs().max() < 1e-5
    # noisy layers (fresh noise per call: compare with the same generator state)
    to_factorized_noisy(q, sigma_scale=0.5)
    monkeypatch.setenv("B2RL_LINEAR", "tcgen05")
    torch.manual_seed(1)
    n_before = len(calls)
    o1 = q(x).q_values
    assert len(calls) == n_before + 3
    monkeypatch.setenv("B2RL_LINEAR", "cublas")
    torch.manual_seed(1)
    o2 = q(x).q_values
    assert (o1 - o2).abs().max() < 1e-5
