"""CPU: the index tables behind the implicit-GEMM convolutions (pfrl_b200/ops/conv.py) describe
exactly torch's convolution, its input gradient (per stride phase) and its weight gradient.

The gather rule of csrc/gemm.cu -- element (row, k) at row_off[row] + k_off[k], present iff
0 <= y + dy < y_limit and 0 <= x + dx < x_limit when the operand carries coordinates -- and the
scatter rule of its epilogue are emulated in numpy (fp64) and compared with
torch.nn.functional.conv2d / autograd on the layer shapes of the Atari nets
(pfrl/nn/atari_cnn.py:30-44) and on ragged ones.  No GPU, no library call: host logic only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pfrl_b200.ops.conv import ConvGeometry, _choice
from pfrl_b200.ops.linear import worth_it


def _operand(data, tab, rows, K):
    d = data.reshape(-1).double().numpy()
    ro = tab["row_off"].numpy().astype(np.int64)[:rows]
    ko = tab["k_off"].numpy().astype(np.int64)
    assert ko.shape[0] % 32 == 0 and ko.shape[0] >= K  # padded for the 32-wide table prefetch
    idx = ro[:, None] + ko[None, :K]
    ok = np.ones_like(idx, dtype=bool)
    if tab["row_yx"] is not None:
        ryx = tab["row_yx"].numpy().astype(np.int64)[:rows]
        kyx = tab["k_yx"].numpy().astype(np.int64)[:K]

        def lo16(v):
            v = v & 0xFFFF
            return np.where(v >= 0x8000, v - 0x10000, v)

        yy = (ryx & 0xFFFF)[:, None] + lo16(kyx)[None, :]
        xx = (ryx >> 16)[:, None] + (kyx >> 16)[None, :]
        yl, xl = tab["limits"]
        ok = (yy >= 0) & (yy < yl) & (xx >= 0) & (xx < xl)
    assert idx[ok].min() >= 0 and idx[ok].max() < d.size  # every present element is in bounds
    return np.where(ok, d[np.where(ok, idx, 0)], 0.0)


def _scatter(C, prod, out):
    rows = prod.c_row.numpy().astype(np.int64)
    for n in range(prod.N):
        out[rows + n * prod.c_stride] = C[:, n]


@pytest.mark.parametrize("B,IC,H,W,OC,KH,KW,s", [
    (3, 4, 20, 20, 6, 4, 4, 2),    # conv2-like
    (2, 5, 9, 9, 7, 3, 3, 1),      # conv3-like
    (2, 4, 28, 28, 5, 8, 8, 4),    # conv1-like (16 stride phases)
    (2, 3, 11, 13, 5, 3, 3, 2),    # odd sizes whose windows still cover every pixel
    (2, 3, 12, 14, 5, 3, 3, 2),    # remainder rows / columns that no window covers
    (2, 2, 9, 9, 3, 2, 2, 3),      # stride > kernel: some input pixels get no gradient
])
def test_tables_describe_conv_forward_dgrad_wgrad(B, IC, H, W, OC, KH, KW, s):
    g = ConvGeometry(B, IC, H, W, OC, KH, KW, s, "cpu")
    gen = torch.Generator().manual_seed(B + H)
    x = torch.randn(B, IC, H, W, dtype=torch.float64, generator=gen, requires_grad=True)
    w = torch.randn(OC, IC, KH, KW, dtype=torch.float64, generator=gen, requires_grad=True)
    y = F.conv2d(x, w, stride=s)
    gy = torch.randn(y.shape, dtype=torch.float64, generator=gen)
    gx, gw = torch.autograd.grad(y, (x, w), gy)

    out = np.zeros(y.numel())
    _scatter(_operand(x.detach(), g.fwd.a, g.fwd.M, g.fwd.K) @ w.detach().reshape(OC, -1).numpy().T,
             g.fwd, out)
    np.testing.assert_allclose(out.reshape(y.shape), y.detach().numpy(), atol=1e-12)

    out = np.zeros(x.numel())
    for p in g.dg:
        _scatter(_operand(gy, p.a, p.M, p.K) @ _operand(w.detach(), p.b, p.N, p.K).T, p, out)
    np.testing.assert_allclose(out.reshape(x.shape), gx.numpy(), atol=1e-12)
    assert len(g.dg) <= s * s and g.dg_covers_input == (s <= min(KH, KW))

    out = np.zeros(w.numel())
    _scatter(_operand(x.detach(), g.wg.a, g.wg.M, g.wg.K) @ _operand(gy, g.wg.b, g.wg.N, g.wg.K).T,
             g.wg, out)
    np.testing.assert_allclose(out.reshape(w.shape), gw.numpy(), atol=1e-12)


def test_default_policy_sends_products_where_they_measured_faster(monkeypatch):
    monkeypatch.delenv("B2RL_LINEAR", raising=False)
    monkeypatch.delenv("B2RL_CONV", raising=False)
    assert worth_it(512, 1024, 3136) and worth_it(512, 3136, 1024) and worth_it(1024, 3136, 512)
    assert worth_it(32, 512, 3136)                       # DQN head at B = 32
    assert worth_it(512, 918, 512) and worth_it(918, 512, 512)  # advantage head fwd, dW
    assert not worth_it(512, 512, 918) and not worth_it(512, 51, 512)  # its dX; the value head
    assert _choice(2, 32) == (True, False, False) and _choice(2, 512) == (False, False, True)
    assert _choice(1, 32) == (True, False, False) and _choice(1, 512) == (True, False, True)
    monkeypatch.setenv("B2RL_CONV", "tcgen05")
    monkeypatch.setenv("B2RL_LINEAR", "cublas")
    assert _choice(1, 32) == (True, True, True) and not worth_it(512, 1024, 3136)
