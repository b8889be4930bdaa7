"""K10: the convolutions of the Nature trunk as implicit GEMMs on the tensor cores
(ops/conv.py over b2rl_gemm_tf32x3_ex) against torch's fp64 convolution.

Tolerance: 1e-5 of the largest magnitude of the fp64 result (the 3xTF32 split keeps fp32-level
accuracy; cuDNN's own fp32 error on the same inputs is printed next to it).  Shapes: the
4x4/2 and 3x3/1 layers at B = 32 and B = 512 (pfrl/nn/atari_cnn.py:30-44), the 8x8/4 first
layer on f32 and on raw uint8 frames, and small ragged cases."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

LAYERS = [
    # B, IC, H, W, OC, K, stride
    (32, 32, 20, 20, 64, 4, 2),
    (512, 32, 20, 20, 64, 4, 2),
    (32, 64, 9, 9, 64, 3, 1),
    (512, 64, 9, 9, 64, 3, 1),
    (32, 4, 84, 84, 32, 8, 4),
    (9, 3, 11, 13, 5, 3, 2),      # ragged: odd sizes, stride 2, windows cover every pixel
    (9, 3, 12, 14, 5, 3, 2),      # stride 2 with a remainder: the last row and column unread
    (8, 2, 9, 9, 3, 2, 3),        # stride > kernel: input gradient pixels zero-filled
    (8, 2, 7, 7, 3, 2, 1),
]


def _rel(got, want):
    return float((got.double() - want).abs().max() / want.abs().max())


@pytest.mark.parametrize("B,IC,H,W,OC,K,s", LAYERS)
def test_conv_forward_dgrad_wgrad_vs_fp64(B, IC, H, W, OC, K, s):
    from pfrl_b200.ops.conv import geometry

    g = torch.Generator(device="cuda").manual_seed(B + IC + H)
    x = torch.randn(B, IC, H, W, device="cuda", generator=g)
    w = torch.randn(OC, IC, K, K, device="cuda", generator=g) * 0.1
    b = torch.randn(OC, device="cuda", generator=g)
    geo = geometry(B, IC, H, W, OC, K, K, s, "cuda:0")
    y = geo.forward(x, w, b)
    x64, w64, b64 = (t.double().requires_grad_() for t in (x, w, b))
    y64 = F.conv2d(x64, w64, b64, stride=s)
    gy = torch.randn(y64.shape, device="cuda", generator=g)
    gx64, gw64 = torch.autograd.grad(y64, (x64, w64), gy.double())
    torch.backends.cudnn.allow_tf32 = False
    y32 = F.conv2d(x, w, b, stride=s)
    print(f"[conv {B}x{IC}x{H}x{W} -> {OC} k{K} s{s}] fwd rel {_rel(y, y64.detach()):.2e} "
          f"(cuDNN fp32 {_rel(y32, y64.detach()):.2e})")
    assert y.shape == y64.shape
    assert _rel(y, y64.detach()) < 1e-5
    gx = geo.dgrad(gy, w)
    gw = geo.wgrad(x, gy)
    print(f"    dgrad rel {_rel(gx, gx64):.2e}  wgrad rel {_rel(gw, gw64):.2e}")
    assert _rel(gx, gx64) < 1e-5
    assert _rel(gw, gw64) < 1e-5
    # relu epilogue
    yr = geo.forward(x, w, b, relu=True)
    assert torch.equal(yr, torch.relu(y))


def test_conv1_on_raw_uint8_frames():
    from pfrl_b200.ops.conv import geometry

    g = torch.Generator(device="cuda").manual_seed(3)
    xb = torch.randint(0, 256, (64, 4, 84, 84), dtype=torch.uint8, device="cuda", generator=g)
    w = torch.randn(32, 4, 8, 8, device="cuda", generator=g) * 0.05
    b = torch.randn(32, device="cuda", generator=g)
    scale = float(torch.tensor(1.0 / 255.0, dtype=torch.float32))
    geo = geometry(64, 4, 84, 84, 32, 8, 8, 4, "cuda:0")
    y = geo.forward(xb, w, b, scale=scale)
    xf = xb.to(torch.float32) * scale
    y64 = F.conv2d(xf.double(), w.double(), b.double(), stride=4)
    assert _rel(y, y64) < 1e-5
    gy = torch.randn(y.shape, device="cuda", generator=g)
    gw = geo.wgrad(xb, gy, scale=scale)
    w64 = w.double().requires_grad_()
    (gw64,) = torch.autograd.grad(F.conv2d(xf.double(), w64, None, stride=4), w64, gy.double())
    assert _rel(gw, gw64) < 1e-5


@pytest.mark.parametrize("policy", ["auto", "tcgen05"])
def test_tcconv2d_module_autograd_matches_cudnn(monkeypatch, policy):
    from pfrl_b200.ops.conv import TCConv2d

    monkeypatch.setenv("B2RL_CONV", policy)
    torch.manual_seed(0)
    m = TCConv2d(32, 64, 4, stride=2).cuda()
    x = torch.randn(64, 32, 20, 20, device="cuda", requires_grad=True)
    y = m(x)
    gy = torch.randn_like(y)
    gx, gw, gb = torch.autograd.grad(y, (x, m.weight, m.bias), gy)
    torch.backends.cudnn.allow_tf32 = False
    y2 = F.conv2d(x, m.weight, m.bias, stride=2)
    gx2, gw2, gb2 = torch.autograd.grad(y2, (x, m.weight, m.bias), gy)
    for a, b_ in ((y, y2), (gx, gx2), (gw, gw2), (gb, gb2)):
        assert float((a - b_).abs().max() / b_.abs().max()) < 1e-5
