"""GPU: every path of the 3xTF32 tensor-core product (csrc/gemm.cu) and of the implicit-GEMM
convolutions (ops/conv.py), element by element against an fp64 product, with the error bound
derived here.

Bound.  With U = 2**-24 (the fp32 unit roundoff), every element of C = A . B^T (+ bias) obeys

    |c - c64| <= [EPS_SPLIT + S * EPS_ACC + (splits + 1) * U] * (|A| . |B|^T)[m, n]
                 + U * |bias[n]|

* EPS_SPLIT = 3 * 2**-22 + U.  x = hi + lo + r with hi = rn_tf32(x), lo = rn_tf32(x - hi):
  |lo| <= 2**-11 |x| and |r| <= 2**-11 |x - hi| <= 2**-22 |x|.  The kernel drops lo.lo
  (<= 2**-22 |a b|) and both residues r_a b, a r_b (<= 2**-22 |a b| each); the products of
  TF32 numbers are exact.
* S = 4 * kb_per_split is the number of 8-deep k steps one split accumulates; each step adds
  eight products to the running fp32 accumulator.  EPS_ACC = 2**-21 is an ASSUMPTION about the
  tensor core: one k8 step of `wgmma ... .f32.tf32.tf32` adds at most 2**-21 of the magnitudes
  it has summed so far (truncation when the nine addends are aligned and when the sum is
  normalised).  The partial magnitudes never exceed (|A| . |B|^T)[m, n].  Each case prints the
  observed per-step error (`eps/step`) so that the assumption is checked on the hardware.
  Truncation is biased: on same-sign data the error grows linearly in S instead of cancelling.
  On an H100 80GB HBM3 (700 W power limit) the same-sign cases reach about 2**-24 per step
  (err / (|A| . |B|^T) = 5.9e-5 at S = 1024, K = 8192 in one split), an eighth of EPS_ACC;
  random-sign products with K >= 512 stay below 2**-26 per step.
* (splits + 1) * U: the epilogue's acc + cor, the splits - 1 additions of the split-K reduce
  and the bias addition, each at most U of a partial magnitude; the bias addition adds U |bias|.
* relu is 1-Lipschitz, so the same bound holds after it.

splits and kb_per_split come from a restatement of plan_splits, which the test checks against
the split count the library reports (b2rl_gemm_workspace_bytes / (4 M N)) on this device.
Random-sign products also keep the older yardstick: at most 4x cuBLAS' own fp32 error.

Convolutions use the same bound with |A| . |B|^T replaced by the convolution of the
magnitudes (F.conv2d(|x|, |w|), and the matching input- and weight-gradient products of |gy|),
S and splits taken from the plan of each product.  conv1's FFMA kernel (csrc/conv.cu) starts
from the bias and rounds 256 fmaf: |y - y64| <= 258 U (F.conv2d(|x|, |w|) + |bias|).  Products
that the module policies may route to cuBLAS fp32 are held to the larger of this bound and the
classical fp32 dot-product bound (K + 2) U (|A| . |B|^T); to cuDNN fp32, four times the classical
bound (its transform algorithms round a few more times per term).

Non-finite inputs: a NaN (torch's 0x7fc00000) or Inf in row i of A or column j of B makes
exactly that row / column of C non-finite (Inf or NaN; csrc/gemm.cu, split_tf32).  The NaN
0x7fffffff that CUDA's own arithmetic produces is rounded to zero by the split and drops out
of the product; the strict xfail below pins that known defect.

Extents.  Dense operands are views into buffers filled with NaN (rows past the operand, `ld`
padding, columns past K); C is a view into a buffer whose padding and extra rows hold a
sentinel bit pattern that must come back unchanged; the split-K workspace starts as NaN.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
EPS_SPLIT = 3 * 2.0 ** -22 + U
EPS_ACC = 2.0 ** -21  # assumed per-k8-step accumulation error of the tensor core (see above)
BM, BK = 128, 32      # output tile rows and k block depth of k_gemm_tf32x3
SENTINEL = 0x7FA5A5A5  # a NaN payload no float operation produces


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def lib():
    from pfrl_b200 import _lib

    return _lib.load()


def n_tile(N):
    return 32 if N <= 32 else 64 if N <= 64 else 128


def plan(M, N, K):
    """(splits, kb_per_split, bn) of a product, as csrc/gemm.cu plans it on this device; the
    split count is checked against the library's."""
    bn = n_tile(N)
    tiles = -(-M // BM) * -(-N // bn)
    kb = -(-K // BK)
    s = max(1, min(sms() // tiles, kb // 4))
    per = -(-kb // s)
    s = -(-kb // per)
    need = lib().b2rl_gemm_workspace_bytes(M, N, K)
    assert (need // (4 * M * N) if need else 1) == s, (M, N, K, need, s)
    return s, per, bn


def reduce_kernel(M, N, splits):
    if splits == 1:
        return None
    return "k_gemm_reduce" if M * N >= 65536 or splits <= 8 else "k_gemm_reduce_deep"


def split_class(M, N, splits):
    if splits == 1:
        return "1"
    if splits <= 8:
        return "2-8"
    return ">8 small" if M * N < 65536 else ">8 large"


def coef(splits, per):
    return EPS_SPLIT + 4 * per * EPS_ACC + (splits + 1) * U


def check(what, got, want, ab, c, bias_abs=None, S=None, extra_ok=None):
    """|got - want| <= c * ab (+ U |bias|) element-wise; prints the worst ratio to the bound
    and the per-step error it implies.  extra_ok: elements not checked (planted non-finite)."""
    got, want, ab = got.double(), want.double(), ab.double()
    bound = c * ab
    if bias_abs is not None:
        bound = bound + U * bias_abs.double()
    err = (got - want).abs()
    ok = err <= bound
    if extra_ok is not None:
        ok |= extra_ok
    sel = ~extra_ok if extra_ok is not None else torch.ones_like(ok)
    ratio = float((err / bound.clamp_min(1e-300))[sel].max()) if bool(sel.any()) else 0.0
    rel = float((err / ab.clamp_min(1e-300))[sel].max()) if bool(sel.any()) else 0.0
    line = f"[{what}] worst err / bound {ratio:.3e}, err / (|A||B|) {rel:.3e}"
    if S:
        line += f", eps/step <= {rel / S:.3e} (assumed {EPS_ACC:.3e})"
    print(line)
    if not bool(ok.all()):
        i = int(torch.nonzero(~ok.reshape(-1))[0])
        raise AssertionError("%s: %d of %d outside the bound; first at %d: got %r, want %r, "
                             "bound %r" % (what, int((~ok).sum()), ok.numel(), i,
                                           got.reshape(-1)[i].item(), want.reshape(-1)[i].item(),
                                           bound.reshape(-1)[i].item()))
    return ratio


# ---------------------------------------------------------------------------
# Dense products through b2rl_gemm_tf32x3
# ---------------------------------------------------------------------------
def fill(kind, shape, g):
    if kind == "randn":
        return torch.randn(shape, device=DEV, generator=g)
    if kind == "pos":
        return torch.rand(shape, device=DEV, generator=g)
    if kind == "spread":  # same sign, magnitudes over 2**-20 .. 2**20
        e = torch.rand(shape, device=DEV, generator=g) * 40 - 20
        return torch.rand(shape, device=DEV, generator=g) * torch.exp2(e)
    raise ValueError(kind)


def operand(data, layout):
    """`data` [rows, cols] copied into a view of a NaN-filled buffer: extra rows, `ld`
    padding, and for layouts o1 / o2 / o3 a start 1-3 floats past 16-byte alignment and
    for `odd` an odd ld (both make the kernel take 4-byte loads)."""
    rows, cols = data.shape
    off = {"o1": 1, "o2": 2, "o3": 3}.get(layout, 0)
    if layout == "odd":
        ld = cols + 1 if cols % 2 == 0 else cols + 2
    else:
        ld = -(-cols // 4) * 4 + 4
    buf = torch.full((off + (rows + 2) * ld,), float("nan"), device=DEV)
    view = buf[off:off + rows * ld].view(rows, ld)[:, :cols]
    view.copy_(data)
    return view, ld


def output(M, N, scalar):
    """C: a view of a sentinel-filled buffer, ldc padded past N to a multiple of 4 (float4
    epilogue, with a ragged tail when N % 4 != 0), or 1 float past alignment (scalar epilogue)."""
    ldc = -(-N // 4) * 4 + 4
    off = 1 if scalar else 0
    buf = torch.full((off + (M + 2) * ldc,), SENTINEL, dtype=torch.int32, device=DEV)
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[off:off + M * ldc].view(M, ldc)[:, :N] = False
    view = buf.view(torch.float32)[off:off + M * ldc].view(M, ldc)[:, :N]
    return buf, outside, view, ldc


def run_gemm(a_st, lda, a_mn, b_st, ldb, b_mn, bias, relu, c, ldc, M, N, K, ws):
    from pfrl_b200 import _lib

    _lib.check(lib().b2rl_gemm_tf32x3(
        ctypes.c_void_p(a_st.data_ptr()), lda, int(a_mn),
        ctypes.c_void_p(b_st.data_ptr()), ldb, int(b_mn),
        None if bias is None else ctypes.c_void_p(bias.data_ptr()), int(relu),
        ctypes.c_void_p(c.data_ptr()), ldc, M, N, K,
        None if ws is None else ctypes.c_void_p(ws.data_ptr()),
        0 if ws is None else ws.numel() * 4,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))


def make_ab(M, N, K, data, g):
    """Logical A [M, K], B [N, K] (fp32).  `cancel`: even rows of A are [x, x] against
    columns of B that are [y, -y], so c64 = 0 there while |A| . |B|^T is large."""
    if data != "cancel":
        return fill(data, (M, K), g), fill(data, (N, K), g)
    a, b = fill("randn", (M, K), g), fill("randn", (N, K), g)
    h = K // 2
    a[::2, h:2 * h] = a[::2, :h]
    b[:, h:2 * h] = -b[:, :h]
    return a, b


def dense_case(M, N, K, a_mn, b_mn, epi, layout, data, seed, bias_off=0, poison=None):
    """One product through the C ABI; returns what the checks need."""
    g = gen(seed)
    a, b = make_ab(M, N, K, data, g)
    if poison:
        poison(a, b)
    a_st, lda = operand(a.t() if a_mn else a, layout if layout != "cs" else "v")
    b_st, ldb = operand(b.t() if b_mn else b, layout if layout != "cs" else "v")
    bias = None
    if "b" in epi:
        bbuf = torch.full((N + 8,), float("nan"), device=DEV)
        bias = bbuf[bias_off:bias_off + N]
        bias.copy_(torch.randn(N, device=DEV, generator=g) * 4)
    cbuf, outside, c, ldc = output(M, N, layout == "cs")
    splits, per, bn = plan(M, N, K)
    need = lib().b2rl_gemm_workspace_bytes(M, N, K)
    ws = torch.full((need // 4,), float("nan"), device=DEV) if need else None
    before = cbuf.clone()
    run_gemm(a_st, lda, a_mn, b_st, ldb, b_mn, bias, "r" in epi, c, ldc, M, N, K, ws)
    torch.cuda.synchronize()
    assert torch.equal(cbuf[outside], before[outside]), "wrote outside C[:M, :N]"
    first = c.clone()
    run_gemm(a_st, lda, a_mn, b_st, ldb, b_mn, bias, "r" in epi, c, ldc, M, N, K, ws)
    assert torch.equal(c.view(torch.int32), first.view(torch.int32)), "not deterministic"
    a64, b64 = a.double(), b.double()
    ref = a64 @ b64.t()
    if bias is not None:
        ref = ref + bias.double()
    if "r" in epi:
        ref = ref.clamp_min(0)
    ab = a64.abs() @ b64.abs().t()
    babs = None if bias is None else bias.double().abs().expand(M, N)
    return dict(c=first, ref=ref, ab=ab, babs=babs, splits=splits, per=per, bn=bn, a=a, b=b,
                bias=bias)


# M, N, K, a_mn, b_mn, epilogue (b: bias, r: relu), layout, data
#   layout: v = aligned, ld padded; o1-o3 = operands 1-3 floats off alignment; odd = odd ld;
#           cs = C one float off alignment (scalar epilogue)
DENSE = [
    # the Rainbow / DQN layers and their backward products
    (512, 1024, 3136, False, False, "br", "v", "randn"),   # main_stream forward
    (512, 3136, 1024, False, True, "", "v", "randn"),      # main_stream dX
    (1024, 3136, 512, True, True, "", "v", "randn"),       # main_stream dW
    (512, 918, 512, False, False, "b", "v", "randn"),      # a_stream forward
    (512, 51, 512, False, False, "r", "odd", "randn"),     # v_stream forward
    (32, 512, 3136, False, False, "br", "v", "randn"),     # DQN head at B = 32
    (256, 256, 8192, False, False, "", "v", "randn"),      # deep K, M N = 65536
    # large batches: one split, bias / relu in the kernel's own epilogue
    (4096, 1024, 3136, False, False, "br", "v", "randn"),  # float4
    (4096, 918, 3136, True, False, "b", "v", "randn"),     # float4 with a ragged tail
    (8192, 129, 1024, False, True, "r", "cs", "randn"),    # scalar
    (8576, 33, 1024, True, True, "br", "cs", "randn"),     # scalar, bn = 64
    # small K: one k block or less, operands off alignment
    (127, 65, 1, False, False, "b", "o1", "randn"),
    (128, 64, 3, True, False, "r", "o2", "randn"),
    (129, 32, 4, False, True, "br", "o3", "randn"),
    (1, 1, 31, True, True, "", "odd", "randn"),
    (1, 16, 32, False, False, "b", "cs", "randn"),
    (129, 128, 33, True, True, "br", "v", "randn"),
    (127, 918, 33, False, True, "r", "o1", "randn"),
    # same-sign data, one split and split
    (4096, 1024, 1024, False, False, "", "v", "pos"),
    (4096, 1024, 3136, False, True, "", "v", "spread"),
    (4096, 1024, 8192, False, False, "b", "v", "pos"),
    (512, 1024, 1024, False, False, "", "v", "pos"),
    (512, 1024, 3136, True, True, "", "v", "spread"),
    (256, 256, 8192, False, False, "", "v", "pos"),
    (32, 512, 3136, False, False, "", "v", "spread"),
    # cancelling rows: c64 = 0, |A| . |B|^T large
    (512, 3136, 1024, False, True, "", "v", "cancel"),
    (256, 256, 8192, False, False, "b", "v", "cancel"),
]


@pytest.mark.parametrize("M,N,K,a_mn,b_mn,epi,layout,data", DENSE)
def test_gemm_every_path_vs_fp64(M, N, K, a_mn, b_mn, epi, layout, data):
    r = dense_case(M, N, K, a_mn, b_mn, epi, layout, data, seed=M * 7 + N * 3 + K)
    c = r["c"]
    assert torch.isfinite(c).all(), "NaN from outside the operands' extents"
    S = 4 * r["per"]
    what = (f"gemm {M}x{N}x{K} mn={int(a_mn)}{int(b_mn)} {epi or '-'} {layout} {data} "
            f"splits={r['splits']} S={S} bn={r['bn']}")
    check(what, c, r["ref"], r["ab"], coef(r["splits"], r["per"]), r["babs"], S)
    if data == "randn" and K >= 1024:
        old = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            c32 = F.linear(r["a"], r["b"], r["bias"])
        finally:
            torch.backends.cuda.matmul.allow_tf32 = old
        if "r" in epi:
            c32 = c32.clamp_min(0)
        e_ours = float((c.double() - r["ref"]).abs().max())
        e_cublas = float((c32.double() - r["ref"]).abs().max())
        print(f"    max err {e_ours:.3e}, cuBLAS fp32 {e_cublas:.3e}")
        assert e_ours <= 4 * e_cublas + 1e-6


NONFINITE = [  # M, N, K, a_mn, b_mn: one shape per split class
    (4096, 1024, 1024, False, False),
    (512, 1024, 3136, True, False),
    (32, 512, 3136, False, True),
    (256, 256, 8192, True, True),
]


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", NONFINITE)
def test_gemm_nonfinite_stays_in_its_row_and_column(M, N, K, a_mn, b_mn):
    """NaN / Inf in row i of A or column j of B make exactly row i / column j of C
    non-finite; no tile or split bleeds into another."""
    rows, col = (3, M - 2), N // 2 + 1

    def poison(a, b):
        a[rows[0], K // 3] = float("nan")
        a[rows[1], K - 1] = float("inf")
        b[col, 0] = -float("inf")

    r = dense_case(M, N, K, a_mn, b_mn, "b", "v", "randn", seed=M + N + K, poison=poison)
    c = r["c"]
    planted = torch.zeros_like(c, dtype=torch.bool)
    planted[list(rows)] = True
    planted[:, col] = True
    assert not torch.isfinite(c[planted]).any()
    assert torch.isfinite(c[~planted]).all()
    a, b = r["a"].clone(), r["b"].clone()
    a[~torch.isfinite(a)] = 0
    b[~torch.isfinite(b)] = 0
    a64, b64 = a.double(), b.double()
    bias = r["babs"]  # |bias|; the value itself is in ref
    ref = torch.where(planted, 0.0, r["ref"])
    ab = a64.abs() @ b64.abs().t()
    check(f"nonfinite {M}x{N}x{K} splits={r['splits']}", torch.where(planted, 0.0, c.double()),
          ref, ab, coef(r["splits"], r["per"]), bias, extra_ok=planted)


@pytest.mark.xfail(strict=True, reason="split_tf32 rounds the NaN 0x7fffffff to -0 (its "
                   "rounding carry reaches the sign bit); a per-element test costs 5-7%")
def test_gemm_nan_0x7fffffff_propagates():
    def poison(a, b):
        a[5, 7] = torch.tensor(0x7FFFFFFF, dtype=torch.int32).view(torch.float32)

    r = dense_case(128, 64, 64, False, False, "", "v", "randn", seed=9, poison=poison)
    assert torch.isnan(r["c"][5]).all()


@pytest.mark.parametrize("off", [1, 2, 3])
def test_gemm_unaligned_bias_on_the_float4_epilogue(off):
    """A bias that is a view at a float offset not a multiple of 4 (a flat parameter buffer)
    on the one-split float4 path: it is read as scalars, not as a misaligned float4."""
    M, N, K = 4096, 1024, 3136
    r = dense_case(M, N, K, False, False, "br", "v", "randn", seed=11 + off, bias_off=off)
    assert r["splits"] == 1
    check(f"unaligned bias +{off}", r["c"], r["ref"], r["ab"], coef(1, r["per"]), r["babs"])


def test_linear_gemm_with_unaligned_bias_view():
    from pfrl_b200.ops.linear import gemm

    g = gen(12)
    a = torch.randn(4096, 3136, device=DEV, generator=g)
    w = torch.randn(1024, 3136, device=DEV, generator=g)
    flat = torch.randn(1024 * 3 + 1, device=DEV, generator=g)
    bias = flat[1:1 + 1024]  # as torch.nn.utils.vector_to_parameters leaves it
    assert bias.data_ptr() % 16 == 4
    c = gemm(a, w, bias=bias, relu=True)
    splits, per, _ = plan(4096, 1024, 3136)
    a64, w64 = a.double(), w.double()
    check("linear.gemm unaligned bias", c, (a64 @ w64.t() + bias.double()).clamp_min(0),
          a64.abs() @ w64.abs().t(), coef(splits, per), bias.double().abs().expand(4096, 1024))


def test_gemm_cases_cover_every_path():
    """Which split count, reduce kernel, bn and epilogue a case takes is decided at run time
    from the SM count; the case lists above must reach every one of them on this device."""
    seen = set()
    for M, N, K, a_mn, b_mn, epi, layout, data in DENSE:
        splits, _, bn = plan(M, N, K)
        seen.add(("split", split_class(M, N, splits)))
        seen.add(("reduce", reduce_kernel(M, N, splits)))
        seen.add(("bn", bn))
        seen.add(("orient", a_mn, b_mn))
        path = "kernel" if splits == 1 else "reduce"
        seen.add(("epilogue", path, epi))
        if splits == 1:
            store = "scalar" if layout == "cs" else "float4" if N % 4 == 0 else "float4 tail"
            seen.add(("store", store))
        if layout in ("o1", "o2", "o3", "odd"):
            seen.add(("unaligned operands",))
        if data in ("pos", "spread"):
            seen.add(("same sign", "1" if splits == 1 else "split", K))
    for M, N, K, *_ in NONFINITE:
        seen.add(("nonfinite", split_class(M, N, plan(M, N, K)[0])))
    assert plan(4096, 1024, 3136)[0] == 1  # the unaligned-bias cases take the float4 epilogue
    want = {("split", s) for s in ("1", "2-8", ">8 small", ">8 large")}
    want |= {("reduce", k) for k in ("k_gemm_reduce", "k_gemm_reduce_deep")}
    want |= {("bn", b) for b in (32, 64, 128)}
    want |= {("orient", x, y) for x in (False, True) for y in (False, True)}
    want |= {("epilogue", p, e) for p in ("kernel", "reduce") for e in ("", "b", "r", "br")}
    want |= {("store", s) for s in ("float4", "float4 tail", "scalar")}
    want |= {("unaligned operands",)}
    want |= {("same sign", p, K) for p in ("1", "split") for K in (1024, 3136, 8192)}
    want |= {("nonfinite", s) for s in ("1", "2-8", ">8 small", ">8 large")}
    missing = want - seen
    print(f"[coverage] {sms()} SMs, {len(seen)} classes reached")
    assert not missing, sorted(map(str, missing))


# ---------------------------------------------------------------------------
# Convolutions through ConvGeometry
# ---------------------------------------------------------------------------
def _conv_abs(x, w, gy, s):
    """fp64 magnitude products: forward, input gradient, weight gradient."""
    xa, wa, ga = x.double().abs(), w.double().abs(), gy.double().abs()
    return (F.conv2d(xa, wa, stride=s),
            torch.nn.grad.conv2d_input(tuple(x.shape), wa, ga, stride=s),
            torch.nn.grad.conv2d_weight(xa, tuple(w.shape), ga, stride=s))


def _prod_coef(prods):
    c = 0.0
    for p in prods:
        splits, per, _ = plan(p.M, p.N, p.K)
        c = max(c, coef(splits, per))
    return c


CONVS = [
    # B, IC, H, W, OC, K, stride
    (8, 32, 20, 20, 64, 4, 2), (32, 32, 20, 20, 64, 4, 2),     # LargeAtariCNN / Rainbow conv2
    (128, 32, 20, 20, 64, 4, 2), (512, 32, 20, 20, 64, 4, 2),
    (8, 64, 9, 9, 64, 3, 1), (32, 64, 9, 9, 64, 3, 1),         # conv3
    (128, 64, 9, 9, 64, 3, 1), (512, 64, 9, 9, 64, 3, 1),
    (8, 4, 84, 84, 16, 8, 4), (32, 4, 84, 84, 16, 8, 4),       # SmallAtariCNN conv1 (N = 16)
    (128, 4, 84, 84, 16, 8, 4),
    (8, 16, 20, 20, 32, 4, 2), (32, 16, 20, 20, 32, 4, 2),     # SmallAtariCNN conv2
    (128, 16, 20, 20, 32, 4, 2),
    (9, 3, 12, 14, 5, 3, 2),     # (12 - 3) and (14 - 3) odd: a row and a column no window covers
    (8, 2, 9, 9, 3, 2, 3),       # stride > kernel: zero-filled input gradient pixels
    (8, 16, 10, 10, 33, 1, 1),   # 1x1 kernel, OC = 33
    (8, 8, 12, 12, 1, 3, 1),     # OC = 1
    (16, 8, 12, 12, 65, 3, 2),   # OC = 65
    (8, 4, 10, 10, 129, 2, 2),   # OC = 129
]


@pytest.mark.parametrize("B,IC,H,W,OC,K,s", CONVS)
def test_conv_products_vs_fp64_per_element(B, IC, H, W, OC, K, s):
    from pfrl_b200.ops.conv import geometry

    g = gen(B * 31 + IC * 7 + H + OC)
    x = torch.randn(B, IC, H, W, device=DEV, generator=g)
    w = torch.randn(OC, IC, K, K, device=DEV, generator=g) * 0.1
    b = torch.randn(OC, device=DEV, generator=g)
    geo = geometry(B, IC, H, W, OC, K, K, s, "cuda:0")
    x64, w64 = x.double(), w.double()
    y64 = F.conv2d(x64, w64, b.double(), stride=s)
    gy = torch.randn(y64.shape, device=DEV, generator=g)
    gx64 = torch.nn.grad.conv2d_input(tuple(x.shape), w64, gy.double(), stride=s)
    gw64 = torch.nn.grad.conv2d_weight(x64, tuple(w.shape), gy.double(), stride=s)
    ab_y, ab_gx, ab_gw = _conv_abs(x, w, gy, s)
    babs = b.double().abs()[None, :, None, None].expand_as(y64)
    tag = f"conv {B}x{IC}x{H}x{W} -> {OC} k{K} s{s}"
    fwd_splits = plan(geo.fwd.M, geo.fwd.N, geo.fwd.K)[0]

    y = geo.forward(x, w, b)
    check(f"{tag} fwd splits={fwd_splits}", y, y64, ab_y, _prod_coef([geo.fwd]), babs)
    yr = geo.forward(x, w, b, relu=True)
    check(f"{tag} fwd bias+relu", yr, y64.clamp_min(0), ab_y, _prod_coef([geo.fwd]), babs)
    gw = geo.wgrad(x, gy)
    check(f"{tag} wgrad splits={plan(geo.wg.M, geo.wg.N, geo.wg.K)[0]}", gw, gw64, ab_gw,
          _prod_coef([geo.wg]))

    # every input pixel is written by exactly one stride phase (or by none, and then zero)
    hits = torch.zeros(x.shape, dtype=torch.int32, device=DEV)
    gx_phases = torch.zeros(x.shape, dtype=torch.float64, device=DEV)
    for prod in geo.dg:
        out = torch.full(x.shape, float("nan"), device=DEV)
        geo._run(prod, geo._gather(gy, prod.a), geo._gather(w, prod.b), out)
        done = ~torch.isnan(out)
        hits += done.int()
        gx_phases += torch.where(done, out.double(), 0.0)
    assert int(hits.max()) == 1
    assert geo.dg_covers_input == bool((hits == 1).all())
    assert (gx64[hits == 0] == 0).all()
    gx = geo.dgrad(gy, w)
    assert torch.equal(gx.double(), gx_phases)
    check(f"{tag} dgrad ({len(geo.dg)} phases)", gx, gx64, ab_gx, _prod_coef(geo.dg))


@pytest.mark.parametrize("u8", [False, True])
def test_conv1_forward_and_wgrad_at_b512(u8):
    """conv1 8x8/4 at the Rainbow batch: the weight gradient is the deepest product the
    library runs (K = 512 * 400, about 66 splits, k_gemm_reduce_deep)."""
    from pfrl_b200.ops.conv import geometry

    B = 512
    g = gen(40 + u8)
    scale = float(torch.tensor(1.0 / 255.0, dtype=torch.float32))
    if u8:
        xin = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, device=DEV, generator=g)
        xin[0, 0, :2] = 0
        xin[0, 0, 2:4] = 255
        x = xin.to(torch.float32) * scale  # the operand values the kernel forms
    else:
        x = xin = torch.randn(B, 4, 84, 84, device=DEV, generator=g)
    w = torch.randn(32, 4, 8, 8, device=DEV, generator=g) * 0.05
    b = torch.randn(32, device=DEV, generator=g)
    geo = geometry(B, 4, 84, 84, 32, 8, 8, 4, "cuda:0")
    splits = plan(geo.wg.M, geo.wg.N, geo.wg.K)[0]
    assert reduce_kernel(geo.wg.M, geo.wg.N, splits) == "k_gemm_reduce_deep"
    gy = torch.randn(B, 32, 20, 20, device=DEV, generator=g)
    ab_y, _, ab_gw = _conv_abs(x, w, gy, 4)
    y = geo.forward(xin, w, b, scale=scale if u8 else None)
    y64 = F.conv2d(x.double(), w.double(), b.double(), stride=4)
    check(f"conv1 fwd u8={u8}", y, y64, ab_y, _prod_coef([geo.fwd]),
          b.double().abs()[None, :, None, None].expand_as(y64))
    gw = geo.wgrad(xin, gy, scale=scale if u8 else None)
    gw64 = torch.nn.grad.conv2d_weight(x.double(), tuple(w.shape), gy.double(), stride=4)
    check(f"conv1 wgrad u8={u8} splits={splits}", gw, gw64, ab_gw, _prod_coef([geo.wg]),
          S=4 * plan(geo.wg.M, geo.wg.N, geo.wg.K)[1])


# ---------------------------------------------------------------------------
# Modules: each branch of ops.linear.worth_it / ops.conv._choice, conv1's FFMA kernel
# ---------------------------------------------------------------------------
@pytest.fixture
def no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _module_coef(M, N, K):
    """Our bound for the product, or the classical fp32 one if cuBLAS computes it."""
    splits, per, _ = plan(M, N, K)
    return max(coef(splits, per), (K + 2) * U)


def _cudnn_coef(ours, K):
    """Our bound, or 4x the classical one if cuDNN computes it (its transform algorithms,
    e.g. Winograd, carry a few more roundings per term than a plain dot product)."""
    return max(ours, 4 * (K + 2) * U)


@pytest.mark.parametrize("policy,B", [("auto", 32), ("auto", 128), ("auto", 512),
                                      ("tcgen05", 32)])
def test_tclinear_autograd_vs_fp64(monkeypatch, no_tf32, policy, B):
    from pfrl_b200.ops.linear import TCLinear

    monkeypatch.setenv("B2RL_LINEAR", policy)
    torch.manual_seed(B)
    m = TCLinear(3136, 512).cuda()
    x = torch.randn(B, 3136, device=DEV, requires_grad=True)
    y = m(x)
    gy = torch.randn_like(y)
    gx, gw, gb = torch.autograd.grad(y, (x, m.weight, m.bias), gy)
    x64, w64, gy64 = x.detach().double(), m.weight.detach().double(), gy.double()
    tag = f"TCLinear {policy} B={B}"
    check(f"{tag} y", y, x64 @ w64.t() + m.bias.double(), x64.abs() @ w64.abs().t(),
          _module_coef(B, 512, 3136), m.bias.detach().double().abs().expand(B, 512))
    check(f"{tag} gx", gx, gy64 @ w64, gy64.abs() @ w64.abs(), _module_coef(B, 3136, 512))
    check(f"{tag} gw", gw, gy64.t() @ x64, gy64.abs().t() @ x64.abs(), _module_coef(512, 3136, B))
    check(f"{tag} gb", gb, gy64.sum(0), gy64.abs().sum(0), (B + 2) * U)


@pytest.mark.parametrize("policy,B", [("auto", 32), ("auto", 128), ("auto", 512),
                                      ("tcgen05", 32)])
@pytest.mark.parametrize("IC,H,OC,K,s", [(32, 20, 64, 4, 2), (64, 9, 64, 3, 1)])
def test_tcconv2d_autograd_vs_fp64(monkeypatch, no_tf32, policy, B, IC, H, OC, K, s):
    from pfrl_b200.ops.conv import TCConv2d, geometry

    monkeypatch.setenv("B2RL_CONV", policy)
    torch.manual_seed(B + IC)
    m = TCConv2d(IC, OC, K, stride=s).cuda()
    x = torch.randn(B, IC, H, H, device=DEV, requires_grad=True)
    y = m(x)
    gy = torch.randn_like(y)
    gx, gw, gb = torch.autograd.grad(y, (x, m.weight, m.bias), gy)
    x64, w64, gy64 = x.detach().double(), m.weight.detach().double(), gy.double()
    ab_y, ab_gx, ab_gw = _conv_abs(x.detach(), m.weight.detach(), gy, s)
    geo = geometry(B, IC, H, H, OC, K, K, s, "cuda:0")
    kk = IC * K * K
    c_y = _cudnn_coef(_prod_coef([geo.fwd]), kk)
    c_gx = _cudnn_coef(_prod_coef(geo.dg), OC * K * K)
    c_gw = _cudnn_coef(_prod_coef([geo.wg]), geo.wg.K)
    tag = f"TCConv2d {policy} B={B} {IC}->{OC} k{K}s{s}"
    y64 = F.conv2d(x64, w64, m.bias.double(), stride=s)
    check(f"{tag} y", y, y64, ab_y, c_y,
          m.bias.detach().double().abs()[None, :, None, None].expand_as(y64))
    check(f"{tag} gx", gx, torch.nn.grad.conv2d_input(tuple(x.shape), w64, gy64, stride=s),
          ab_gx, c_gx)
    check(f"{tag} gw", gw, torch.nn.grad.conv2d_weight(x64, tuple(w64.shape), gy64, stride=s),
          ab_gw, c_gw)
    n = gy[0, 0].numel() * B
    check(f"{tag} gb", gb, gy64.sum((0, 2, 3)), gy64.abs().sum((0, 2, 3)), (n + 2) * U)


@pytest.mark.parametrize("u8", [False, True])
@pytest.mark.parametrize("n", [1, "2sms+3"])
def test_nature_conv1_ffma_kernel_vs_fp64(u8, n):
    """csrc/conv.cu: 256 fp32 FMAs per output from the bias; n > 2 SMs makes every CTA run
    three images, so the uint8 double buffer turns over."""
    from pfrl_b200.nn.fast_conv import NatureConv1

    n = 2 * sms() + 3 if n == "2sms+3" else n
    torch.manual_seed(n)
    m = NatureConv1().cuda()
    g = gen(50 + n + u8)
    if u8:
        xin = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, device=DEV, generator=g)
        xin[-1, -1, -2:] = 255
        xin[0, 0, :2] = 0
        x = xin.to(torch.float32) * m.input_scale
    else:
        x = xin = torch.randn(n, 4, 84, 84, device=DEV, generator=g)
    with torch.no_grad():
        y = m(xin)
    w64, b64 = m.weight.detach().double(), m.bias.detach().double()
    y64 = F.conv2d(x.double(), w64, b64, stride=4)
    ab = F.conv2d(x.double().abs(), w64.abs(), stride=4) + b64.abs()[None, :, None, None]
    check(f"NatureConv1 u8={u8} n={n}", y, y64, ab, 258 * U)


@pytest.mark.parametrize("u8", [False, True])
def test_nature_conv1_tcgen05_backward(monkeypatch, u8):
    """B2RL_CONV=tcgen05: the weight gradient of both conv1 autograd functions comes from the
    implicit GEMM (from the bytes for uint8)."""
    from pfrl_b200.nn.fast_conv import NatureConv1
    from pfrl_b200.ops.conv import geometry

    monkeypatch.setenv("B2RL_CONV", "tcgen05")
    B = 64
    torch.manual_seed(60 + u8)
    m = NatureConv1().cuda()
    g = gen(60 + u8)
    if u8:
        xin = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, device=DEV, generator=g)
        x = xin.to(torch.float32) * m.input_scale
    else:
        x = xin = torch.randn(B, 4, 84, 84, device=DEV, generator=g)
    y = m(xin)
    gy = torch.randn_like(y)
    gw, gb = torch.autograd.grad(y, (m.weight, m.bias), gy)
    _, _, ab_gw = _conv_abs(x, m.weight.detach(), gy, 4)
    geo = geometry(B, 4, 84, 84, 32, 8, 8, 4, "cuda:0")
    gy64 = gy.double()
    check(f"NatureConv1 tcgen05 wgrad u8={u8}", gw,
          torch.nn.grad.conv2d_weight(x.double(), (32, 4, 8, 8), gy64, stride=4), ab_gw,
          _prod_coef([geo.wg]))
    check(f"NatureConv1 tcgen05 gb u8={u8}", gb, gy64.sum((0, 2, 3)),
          gy64.abs().sum((0, 2, 3)), (B * 400 + 2) * U)
