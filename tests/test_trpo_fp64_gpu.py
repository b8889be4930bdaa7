"""TRPO's policy-update kernels (csrc/trpo.cu) and the fused policy update
(agents/trpo.py ``_policy_kernels``) against fp64, element by element.

Every comparison feeds the fp64 side the fused path's own fp32 inputs, so that a bound
covers the rounding of one stage.  U = 2^-24 (fp32), E = 2^-53 (fp64).  A value that
rounds into fp32's subnormal range carries an absolute error of up to 2^-150 more.

Kernels
* ``k_trpo_fisher``: M u / N per element, M = diag(1/s^2, 2/s^2) (Gaussian) or
  diag(p) - p p^T (categorical, p from the kernel's own re-normalised logits).  The kernel
  works in fp64 and rounds once: |err| <= U |m| + (4K + 16)(2 + max|l|) E (p/N)
  (|u| + sum_j p_j |u_j|), where the second term is the fp64 evaluation of p = e^l and of the
  dot p.u on both sides (|l| <= 200 here, so it is below 2^-30 of its sum).
* CG (``cg_init`` / ``cg_iter``), checked after every launch from the kernel's own state
  before it.  alpha = fp32(r.r / p.Ap): the fp64 dot p.Ap errs by (n + 2) E sum|p Ap|, so
  |alpha' - alpha| <= d_a = |alpha| (U + (n + 2) E sum|p Ap| / |p.Ap|) + tiny.  Then
  x' = fl(x + fl(p alpha')): |err| <= |p| d_a + U |p alpha| + U |x'| (each with a factor
  1 + 4U), the same for r' with Ap.  r.r is fp64 ((n + 2) E r.r); beta = fp32(rr' / rr) is
  formed from the two fp64 values the kernel keeps, so p' = fl(r' + fl(beta' p)) is bounded
  by U (2 |beta p| + |p'|).  The exit flag must equal sqrt(r'.r') < tol unless the two lie
  within (n + 2) E of each other.
* ``k_trpo_cg_step``: dId = fp32(fp64 x.Ax): |err| <= U |dId| + (n + 2) E sum|x Ax|.  The
  scale is fp32(sqrt(2 max_kl / (double(dId) + 1e-8))), which the test evaluates from the
  kernel's dId, and full = fl(scale x) bit for bit.
* ``k_trpo_line_search``: the reference's decision on each candidate (float reads, fp64
  improvement) and theta = fl(theta_old + fl(2^-i full)) bit for bit, theta_old when no
  candidate wins.

The fused policy update, stage by stage, on every policy head (one-hidden-layer tanh MLP,
H = 32).  The fp64 side is the fp64 copy of the policy (the same parameter values) run
through the reference's formulation (``_compute_gain``, ``_hessian_vector_product``).
* Gain, KL, entropy of every candidate: the objective kernel on the fused path's fp32
  distribution parameters against fp64 torch on the same values: U |v| + 2^-36 S, S the
  mean over rows of the magnitudes the fp64 evaluation rounds: |ratio adv| + c |entropy|
  for the gain, and for the KL its terms before they cancel, p_old (|l_old| + |l|) per
  category and ((s_o / s)^2 + t^2 + 1 + |log (s_o / s)^2|) / 2 per Gaussian dimension (the
  fp64 sums over N <= 2048 rows of such terms err by far less than 2^-36 S).
* The flat gradient J^T g and the Fisher-vector product J^T M J v + lambda v: an fp32
  inner product of length k errs by at most k U times the sum of its terms' magnitudes.
  Forward-mode J v runs through inner products of length <= obs + H + 2, the kernel's M u
  rounds once, and the backward to the parameters sums over the N rows and the head's
  outputs, so with C = 2 (N + obs + H + 2 D + 64) + 16 max h^2 / (1 - h^2) (D the
  distribution parameters per row; the 64 covers the elementwise ops; the factor 2 is
  headroom over these first-order counts, which one gradient element of the 18-way softmax
  at N = 1 exceeds by a small factor; fp32's tanh is good to 2 ulp, and its derivative
  1 - h^2, used once in J v and once in J^T, then errs by up to 8 U h^2 / (1 - h^2)
  relative):
  |err(J^T g)| <= C U (|J|^T |g|) + U |J^T g|, |err(F v)| <= C U (|J|^T |M| |J| |v|) +
  2 U (|F v| + lambda |v|).  J is the fp64 Jacobian of the distribution parameters (raw
  logits for the categorical, for which M is shift-invariant), |M| <= diag(p) + p p^T.
  With one hidden layer every parameter has a single path to each output, so |J| is the
  product of the layers' absolute values that the inner-product bound is stated in.
* dId and the full step as for ``k_trpo_cg_step``, on the fused path's own x and F x.
* The decision: the fp64 decision on the fp64 improvements and KLs; the kernel's must equal
  it wherever no candidate up to the fp64 winner lies within its stage bound of a
  threshold.  Each head also gets a planted max_kl two bounds either side of candidate 0's
  KL.
"""
import copy
import math

import numpy as np
import pytest
import torch
from torch import distributions as D
from torch import nn

from pfrl_b200.ops import trpo as fused
from pfrl_b200.utils.modes import no_distribution_validation

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
E = 2.0 ** -53
SUB = 2.0 ** -150  # half the spacing of fp32's subnormals
N_SET = [1, 31, 1023, 1024, 1025, 100000, 2 ** 20 + 3]


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def check(name, got, want, bound):
    """Element-wise |got - want| <= bound (fp64); equal values, NaN included, always pass.
    A failure names the first failing element with its bound."""
    want = torch.as_tensor(want).double().cpu()
    bound = torch.broadcast_to(torch.as_tensor(bound).double().cpu(), want.shape).reshape(-1)
    got, want = torch.as_tensor(got).double().cpu().reshape(-1), want.reshape(-1)
    same = (got == want) | (torch.isnan(got) & torch.isnan(want))
    bad = ~same & ~((got - want).abs() <= bound)
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(
            "%s: element %d of %d (%d failing): got %r, want %r, |err| %.4g > bound %.4g"
            % (name, i, want.numel(), int(bad.sum()), float(got[i]), float(want[i]),
               float((got[i] - want[i]).abs()), float(bound[i])))


def bits_equal(a, b):
    # fresh dense copies: a one-element tensor may keep a zero stride through contiguous()
    a, b = (torch.empty(t.shape, dtype=t.dtype).copy_(t.detach()) for t in (a, b))
    return a.shape == b.shape and a.dtype == b.dtype and \
        torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---------------------------------------------------------------------------- Fisher
def fisher_ref(kind, p, u):
    """fp64 M u / N and the bound of the module docstring, per element."""
    N, A = p[0].shape
    if kind == fused.GAUSSIAN:
        sd = p[1].double()
        w = 1.0 / (N * sd * sd)
        out = [w * u[0].double(), 2.0 * w * u[1].double()]
        return [(m, U * m.abs() + 8 * E * m.abs() + SUB) for m in out]
    z = p[0].double()
    l = z - torch.logsumexp(z, 1, keepdim=True)
    pr = l.exp()
    ud = u[0].double()
    pu = (pr * ud).sum(1, keepdim=True)
    m = pr * (ud - pu) / N
    lmax = torch.where(torch.isfinite(l), l.abs(), torch.zeros(())).amax(1, keepdim=True)
    slop = (4 * A + 16) * (2 + lmax) * E * pr / N * (ud.abs() + (pr * ud.abs()).sum(1, True))
    return [(m, U * m.abs() + slop + SUB)]


def fisher_case(kind, N, A, seed, extreme=False, neg_inf=False):
    g = torch.Generator().manual_seed(seed)
    if kind == fused.GAUSSIAN:
        lsd = (torch.rand(N, A, generator=g) * 18 - 9) if extreme else \
            0.5 * torch.randn(N, A, generator=g)
        p = [torch.randn(N, A, generator=g), torch.exp(lsd)]
        u = [torch.randn(N, A, generator=g), torch.randn(N, A, generator=g)]
        return p, u
    z = torch.randn(N, A, generator=g) * (20.0 if extreme else 1.0)
    if neg_inf and A > 1:
        # -inf at the first category, at the last, and at both
        z[0::3, 0] = -float("inf")
        z[1::3, -1] = -float("inf")
        if A > 2:  # a row of -inf alone has no distribution (torch gives NaN)
            z[2::3, 0] = z[2::3, -1] = -float("inf")
    return [z], [torch.randn(N, A, generator=g)]


def run_fisher(kind, p, u, tangents=None):
    want = fisher_ref(kind, p, u)
    tangents = [t.to(DEV) for t in u] if tangents is None else tangents
    got = fused.fisher(kind, [x.to(DEV) for x in p], tangents)
    for j, (m, bound) in enumerate(want[:len([t for t in tangents if t is not None])]):
        check("fisher kind %d out %d" % (kind, j), got[j], m, bound)
    return got


@pytest.mark.parametrize("N", [1, 255, 256, 257, 5000])
@pytest.mark.parametrize("A", [1, 6, 17])
def test_gaussian_fisher_per_element(N, A):
    run_fisher(fused.GAUSSIAN, *fisher_case(fused.GAUSSIAN, N, A, N * 7 + A))
    p, u = fisher_case(fused.GAUSSIAN, N, A, N * 7 + A + 1, extreme=True)
    run_fisher(fused.GAUSSIAN, p, u)
    # a scale without a gradient: no second tangent, no second output (m1 = NULL)
    for tangents in ([u[0].to(DEV), None], [u[0].to(DEV)]):
        got = run_fisher(fused.GAUSSIAN, p, u, tangents)
        assert len(got) == len(tangents) and (len(got) == 1 or got[1] is None)


@pytest.mark.parametrize("N", [1, 255, 256, 257, 5000])
@pytest.mark.parametrize("K", [2, 18, 257])
def test_categorical_fisher_per_element(N, K):
    run_fisher(fused.CATEGORICAL, *fisher_case(fused.CATEGORICAL, N, K, N * 5 + K))
    run_fisher(fused.CATEGORICAL,
               *fisher_case(fused.CATEGORICAL, N, K, N * 5 + K + 1, extreme=True, neg_inf=True))


# -------------------------------------------------------------------------------- CG
def spd_operator(n, seed):
    """A p = d p + q (q.p), d in [1, 10]: symmetric positive definite, applied in fp32."""
    g = torch.Generator().manual_seed(seed)
    d = (1.0 + 9.0 * torch.rand(n, generator=g)).to(DEV)
    q = (torch.randn(n, generator=g) / math.sqrt(n)).to(DEV)
    return lambda v: d * v + q * torch.dot(q, v)


def cg_checked(A, b, tol, max_iter):
    """Runs cg_init and max_iter cg_iter launches, checking every launch against one fp64
    iteration from the kernel's state before it.  Returns (x, exit iteration or None)."""
    n = b.numel()
    x, r, p, state = fused.cg_init(b)
    b64 = b.double().cpu()
    assert bool((x == 0).all()) and bits_equal(r, b) and bits_equal(p, b)
    st = state.cpu()
    check("cg_init r.r", st[0], (b64 * b64).sum(), (n + 2) * E * (b64 * b64).sum())
    assert float(st[1]) == 0.0
    exit_at = None
    for it in range(1, max_iter + 1):
        x0, r0, p0 = (t.clone() for t in (x, r, p))
        s0 = state.cpu()
        Ap = A(p)
        fused.cg_iter(Ap, x, r, p, state, tol)
        s1 = state.cpu()
        if float(s0[1]) != 0.0:  # converged: nothing moves
            assert bits_equal(x, x0) and bits_equal(r, r0) and bits_equal(p, p0)
            assert bits_equal(s1, s0)
            continue
        x0d, r0d, p0d, Apd = (t.double().cpu() for t in (x0, r0, p0, Ap))
        pAp = p0d * Apd
        pap = pAp.sum()
        alpha = s0[0] / pap
        d_a = abs(alpha) * (U + (n + 2) * E * pAp.abs().sum() / pap.abs()) + 1e-300
        where = "iteration %d of n = %d" % (it, n)
        xw, rw = x0d + alpha * p0d, r0d - alpha * Apd
        check("x, " + where, x, xw,
              (1 + 4 * U) * (p0d.abs() * d_a + U * (p0d * alpha).abs() + U * xw.abs()) + SUB)
        check("r, " + where, r, rw,
              (1 + 4 * U) * (Apd.abs() * d_a + U * (Apd * alpha).abs() + U * rw.abs()) + SUB)
        r1 = r.double().cpu()
        rr1 = (r1 * r1).sum()
        norm = math.sqrt(float(rr1))
        if float(s1[1]) != 0.0:
            exit_at = it
            assert norm < tol or abs(norm - tol) <= (n + 2) * E * norm, (where, norm, tol)
            # the exit leaves p and r.r as they were
            assert bits_equal(p, p0) and float(s1[0]) == float(s0[0])
            continue
        assert not (norm < tol) or abs(norm - tol) <= (n + 2) * E * norm, (where, norm, tol)
        check("r.r, " + where, s1[0], rr1, (n + 2) * E * rr1)
        beta = s1[0] / s0[0]
        pw = r1 + beta * p0d
        check("p, " + where, p, pw,
              (1 + 4 * U) * U * (2 * (beta * p0d).abs() + pw.abs()) + SUB)
    return x, exit_at


@pytest.mark.parametrize("n", N_SET)
def test_cg_every_iteration_against_fp64(n):
    b = torch.randn(n, generator=torch.Generator().manual_seed(n)).to(DEV)
    x, exit_at = cg_checked(spd_operator(n, n + 1), b, 1e-10, 10 if n > 1 else 3)
    assert n == 1 or exit_at is None
    assert bool(torch.isfinite(x).all())


def _torch_cg_exit(A, b, tol, max_iter):
    """The iteration at which the reference's loop returns (None: it ran out)."""
    from pfrl_b200.utils.conjugate_gradient import _conjugate_gradient_torch

    calls = []

    def counted(v):
        calls.append(1)
        return A(v)

    _conjugate_gradient_torch(counted, b, tol, max_iter)
    it = (len(calls) - 1) // 2
    return it if it < max_iter or _torch_exits_last(A, b, tol, max_iter) else None


def _torch_exits_last(A, b, tol, max_iter):
    from pfrl_b200.utils.conjugate_gradient import _conjugate_gradient_torch

    x = _conjugate_gradient_torch(A, b, tol, max_iter)
    return float(torch.norm(b - A(x))) < tol


@pytest.mark.parametrize("n", N_SET)
@pytest.mark.parametrize("m", [1, 5, 10])
def test_cg_exit_at_first_middle_and_last_iteration(n, m):
    """A diagonal system with the m distinct eigenvalues 1 .. m is solved exactly at
    iteration m: the residual there is fp32 round-off, ~1e-7 of |b|, far below
    tol = 1e-5 |b|, while one iteration earlier it is above 1e-4 |b|.  The kernel's exit iteration must be the reference
    loop's, and the launches after it must change nothing."""
    m = min(m, n)
    g = torch.Generator().manual_seed(100 * n + m)
    d = (1.0 + torch.arange(n) % m).float().to(DEV)
    b = torch.randn(n, generator=g).to(DEV)
    tol = 1e-5 * float(torch.norm(b))
    A = lambda v: d * v  # noqa: E731
    x, exit_at = cg_checked(A, b, tol, 10)
    assert exit_at == m
    ref = _torch_cg_exit(A, b, tol, 10)
    assert ref == m, (ref, m)
    check("solution", x, (b / d).double(), 4e-3 * (b / d).double().abs().max())


def test_cg_zero_right_hand_side_gives_nan_like_the_reference():
    from pfrl_b200.utils import conjugate_gradient
    from pfrl_b200.utils.conjugate_gradient import _conjugate_gradient_torch

    for n in (1, 1025):
        A = spd_operator(n, 3)
        b = torch.zeros(n, device=DEV)
        x = conjugate_gradient(A, b, max_iter=4)
        assert bool(torch.isnan(x).all())
        assert bool(torch.isnan(_conjugate_gradient_torch(A, b, max_iter=4)).all())


# --------------------------------------------------------------------------- cg_step
def check_cg_step(x, Ax, max_kl, full, dId, name):
    xd, Axd = x.double().cpu(), Ax.double().cpu()
    prod = xd * Axd
    want = prod.sum()
    dId = float(dId.reshape(()))
    check(name + " dId", dId, want, U * abs(float(want)) + (x.numel() + 2) * E *
          float(prod.abs().sum()))
    scale = np.float32(np.sqrt(2.0 * max_kl / (float(np.float32(dId)) + 1e-8)))
    want_full = torch.from_numpy(scale * x.cpu().numpy()).reshape(-1)
    full = full.reshape(-1).cpu()
    if np.isnan(scale):  # b = 0: NaN (the bit pattern of a NaN is not IEEE's business)
        assert bool(torch.isnan(full).all()), name + " full step"
    else:
        assert bits_equal(full, want_full), name + " full step"


@pytest.mark.parametrize("n", N_SET)
@pytest.mark.parametrize("max_kl", [1e-3, 0.01, 0.05])
def test_cg_step_dId_scale_and_full_step(n, max_kl):
    g = torch.Generator().manual_seed(n)
    x = (torch.randn(n, generator=g) * torch.exp(3 * torch.randn(n, generator=g))).to(DEV)
    Ax = x * (0.5 + torch.rand(n, generator=g)).to(DEV)
    full, dId = fused.cg_step(x, Ax, max_kl)
    check_cg_step(x, Ax, max_kl, full, dId, "n = %d" % n)


# ----------------------------------------------------------------------- line search
def ref_decision(cand, gain0, max_kl):
    """trpo.py _line_search on host floats: the first candidate with a finite gain and
    KL, float(gain) - float(gain0) >= 0 and KL <= max_kl; -1 if none."""
    for i, (g, kl, _) in enumerate(cand):
        g, kl = float(np.float32(g)), float(np.float32(kl))
        improve = g - float(np.float32(gain0))
        if not math.isfinite(g) or not math.isfinite(kl) or improve < 0 or kl > max_kl:
            continue
        return i
    return -1


NAN, INF = float("nan"), float("inf")
REJECT = [[NAN, 0.001, 0], [0.5, INF, 0], [0.5, -INF, 0], [0.5, NAN, 0], [0.05, 0.001, 0],
          [0.5, 0.0101, 0], [INF, 0.001, 0], [-INF, 0.001, 0]]
LS_CASES = {
    "one_winner": ([[0.2, 0.009, 0]], 0),
    "one_nan_gain": ([[NAN, 0.001, 0]], -1),
    "negative_zero_improvement": ([[-0.0, 0.0, 0]], 0),
    "winner_at_0_of_64": ([[0.1, 0.01, 0]] + [[0.2, 0.001, 0]] * 63, 0),
    "winner_at_63": ([REJECT[i % len(REJECT)] for i in range(63)] + [[0.1, 0.001, 0]], 63),
    "none_of_64": ([REJECT[i % len(REJECT)] for i in range(64)], -1),
}


@pytest.mark.parametrize("n", [1, 1000, 256 * 1024, 256 * 1024 + 1, 2 ** 20 + 5])
@pytest.mark.parametrize("case", sorted(LS_CASES))
def test_line_search_decision_and_write(n, case):
    cand, win = LS_CASES[case]
    gain0 = 0.0 if case == "negative_zero_improvement" else 0.1
    max_kl = 0.01
    assert ref_decision(cand, gain0, max_kl) == win
    g = torch.Generator().manual_seed(n)
    theta_old = torch.randn(n, generator=g)
    full = torch.randn(n, generator=g) * torch.exp(4 * torch.randn(n, generator=g))
    theta, rec = fused.line_search(torch.tensor(cand, dtype=torch.float32, device=DEV),
                                   torch.tensor([gain0, 0, 0], device=DEV), max_kl,
                                   theta_old.to(DEV), full.to(DEV))
    rec = rec.cpu().tolist()
    if win < 0:
        assert rec == [0.0, 0.0, 0.0]
        assert bits_equal(theta, theta_old)
        return
    s = 2.0 ** -win
    assert rec == [float(np.float32(cand[win][1])), s, 1.0]
    want = theta_old.numpy() + np.float32(s) * full.numpy()
    assert bits_equal(theta, torch.from_numpy(want))


def test_line_search_refuses_65_candidates():
    cand = torch.zeros(65, 3, device=DEV)
    with pytest.raises(RuntimeError, match="65 candidates"):
        fused.line_search(cand, torch.zeros(3, device=DEV), 0.01,
                          torch.zeros(8, device=DEV), torch.zeros(8, device=DEV))


def test_ops_never_hand_a_kernel_another_dtype():
    """Inputs of another dtype are converted; buffers a kernel writes in place must be
    fp32 already."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1000, generator=g, dtype=torch.float64).to(DEV)
    Ax = 2 * x
    full, dId = fused.cg_step(x, Ax, 0.01)
    full32, dId32 = fused.cg_step(x.float(), Ax.float(), 0.01)
    assert full.dtype == torch.float32 and bits_equal(full, full32) and bits_equal(dId, dId32)
    for dtype in (torch.float64, torch.float16, torch.bfloat16):
        t = torch.zeros(8, device=DEV, dtype=dtype)
        with pytest.raises(AssertionError):
            fused.line_search(torch.zeros(1, 3, device=DEV), torch.zeros(3, device=DEV), 0.01,
                              t.float(), t.float(), theta=t)
        with pytest.raises(AssertionError):
            fused.cg_iter(t, t, t, t, torch.zeros(2, device=DEV, dtype=torch.float64), 1e-10)
    with pytest.raises(AssertionError):
        fused.cg_step(x.cpu(), Ax.cpu(), 0.01)


# ----------------------------------------------------- the fused update, stage by stage
OBS, H = 7, 32
HEADS = ["gauss_diagonal", "gauss_spherical", "gauss_state", "gauss_fixed", "softmax2",
         "softmax18", "softmax_masked"]


class _Mask(nn.Module):
    """Sets logits 1 and 3 to -inf, and logit 0 where the first state entry is positive."""

    def forward(self, z):
        z = z.clone()
        z[:, 1] = z[:, 3] = -float("inf")
        return z.masked_fill((self._s0 > 0)[:, None] & (torch.arange(z.shape[1],
                                                                     device=z.device) == 0),
                             -float("inf"))


class _MaskedMLP(nn.Module):
    def __init__(self, K):
        super().__init__()
        from pfrl_b200.policies import SoftmaxCategoricalHead

        self.body = nn.Sequential(nn.Linear(OBS, H), nn.Tanh(), nn.Linear(H, K))
        self.mask = _Mask()
        self.head = SoftmaxCategoricalHead()

    def raw(self, s):
        self.mask._s0 = s[:, 0]
        return self.mask(self.body(s))

    def forward(self, s):
        return self.head(self.raw(s))


def make_policy(head, seed):
    from pfrl_b200.policies import (GaussianHeadWithDiagonalCovariance,
                                    GaussianHeadWithFixedCovariance,
                                    GaussianHeadWithStateIndependentCovariance,
                                    SoftmaxCategoricalHead)

    torch.manual_seed(seed)
    if head == "softmax_masked":
        return _MaskedMLP(6)
    if head.startswith("softmax"):
        K = int(head[len("softmax"):])
        return nn.Sequential(nn.Linear(OBS, H), nn.Tanh(), nn.Linear(H, K),
                             SoftmaxCategoricalHead())
    A = 6
    if head == "gauss_state":
        return nn.Sequential(nn.Linear(OBS, H), nn.Tanh(), nn.Linear(H, 2 * A),
                             GaussianHeadWithDiagonalCovariance())
    h = GaussianHeadWithFixedCovariance(0.7) if head == "gauss_fixed" else \
        GaussianHeadWithStateIndependentCovariance(A, var_type=head[len("gauss_"):],
                                                   var_param_init=-0.5)
    return nn.Sequential(nn.Linear(OBS, H), nn.Tanh(), nn.Linear(H, A), h)


def raw_params(policy, s):
    """The distribution parameters the Fisher metric acts on, [N, D]: (loc, scale) for a
    Gaussian, the logits before Categorical normalises them."""
    from pfrl_b200.agents.trpo import _distribution_params

    if isinstance(policy, _MaskedMLP):
        return policy.raw(s)
    if isinstance(policy[-1], nn.Module) and type(policy[-1]).__name__ == \
            "SoftmaxCategoricalHead":
        return policy[:-1](s)
    kind, (loc, scale) = _distribution_params(policy(s))
    return torch.cat([loc, scale.expand_as(loc)], 1)


def abs_jacobian_products(pol64, s64, row_vecs, param_vecs, chunk=128):
    """For the fp64 Jacobian J of raw_params (rows [N, D], columns the flat parameters),
    computed in row chunks: [|J|^T |w| for w in row_vecs] and [|J| |v| for v in
    param_vecs] (as [N, D])."""
    names = [n for n, _ in pol64.named_parameters()]
    primals = {n: p.detach() for n, p in pol64.named_parameters()}
    N = s64.shape[0]
    out_t = [0.0] * len(row_vecs)
    out_j = [[] for _ in param_vecs]
    for lo in range(0, N, chunk):
        sc = s64[lo:lo + chunk]
        jac = torch.func.jacrev(
            lambda ps: raw_params_functional(pol64, ps, sc))(primals)
        J = torch.cat([jac[n].reshape(sc.shape[0], -1, primals[n].numel()) for n in names],
                      2).abs()  # [rows, D, P]
        for i, w in enumerate(row_vecs):
            out_t[i] = out_t[i] + torch.einsum("rdp,rd->p", J, w[lo:lo + chunk].abs())
        for i, v in enumerate(param_vecs):
            out_j[i].append(torch.einsum("rdp,p->rd", J, v.abs()))
    return out_t, [torch.cat(o) for o in out_j]


def raw_params_functional(pol64, ps, s):
    return torch.func.functional_call(_RawParams(pol64), {"policy." + k: v for k, v in
                                                          ps.items()}, (s,))


class _RawParams(nn.Module):
    def __init__(self, policy):
        super().__init__()
        self.policy = policy

    def forward(self, s):
        return raw_params(self.policy, s)


class _Spy:
    """Records what the fused update hands to and gets from the kernels' wrappers."""

    def __init__(self, monkeypatch, agent, test_vectors):
        import pfrl_b200.agents.trpo as trpo_mod

        self.cands, self.fvp_out = [], []
        real = dict(gain=fused.gain, objective=fused.objective, cg_step=fused.cg_step,
                    line_search=fused.line_search, cg=trpo_mod.conjugate_gradient,
                    fvp=agent._fisher_vector_product)

        def gain(kind, params, old, *rest):
            self.gain_in = ([p.detach().clone() for p in params], [o.clone() for o in old])
            out = real["gain"](kind, params, old, *rest)
            self.gain_out = out[1].clone()
            return out

        def objective(kind, params, *rest):
            out = real["objective"](kind, params, *rest)
            self.cands.append(([p.detach().clone() for p in params], out.clone()))
            return out

        def fvp_factory(*a):
            f = real["fvp"](*a)
            self.fvp = f
            return f

        def cg(A, b, **kw):
            self.b = b.detach().clone()
            x = real["cg"](A, b, **kw)
            return x

        def cg_step(x, Ax, max_kl):
            # the product for the test vectors, before the parameters are written
            self.fvp_out = [self.fvp(v).detach().clone() for v in test_vectors]
            full, dId = real["cg_step"](x, Ax, max_kl)
            self.cg_step_io = (x.detach().clone(), Ax.detach().clone(), full.clone(),
                               dId.clone())
            return full, dId

        def line_search(cand, gain0, max_kl, theta_old, full_step, theta=None):
            self.ls_in = (cand.clone(), gain0.clone(), theta_old.clone(), full_step.clone())
            theta, record = real["line_search"](cand, gain0, max_kl, theta_old, full_step, theta)
            self.ls_out = (theta.clone(), record.clone())
            return theta, record

        for k, f in (("gain", gain), ("objective", objective), ("cg_step", cg_step),
                     ("line_search", line_search)):
            monkeypatch.setattr(fused, k, f)
        monkeypatch.setattr(trpo_mod, "conjugate_gradient", cg)
        monkeypatch.setattr(agent, "_fisher_vector_product", fvp_factory)


def fp64_objective(agent64, kind, params, old, actions, lp_old, adv_in):
    """gain, KL(old || new), mean entropy in fp64 on fp32 distribution parameters, and the
    per-row magnitudes S_gain, S_kl, S_ent of the sums; d gain / d params."""
    p = [x.double().requires_grad_() for x in params]
    with no_distribution_validation():
        return _fp64_objective(agent64, kind, p, old, actions, lp_old, adv_in)


def _fp64_objective(agent64, kind, p, old, actions, lp_old, adv_in):
    if kind == fused.GAUSSIAN:
        d = D.Independent(D.Normal(p[0], p[1]), 1)
        do = D.Independent(D.Normal(old[0].double(), old[1].double()), 1)
        lp = d.log_prob(actions.double())
    else:
        d, do = D.Categorical(logits=p[0]), D.Categorical(logits=old[0].double())
        lp = d.log_prob(actions)
    ent = d.entropy()
    gain = agent64._compute_gain(log_prob=lp, log_prob_old=lp_old.double(), entropy=ent,
                                 advs=adv_in.double())
    kl_rows = D.kl_divergence(do, d)
    # the KL's terms before they cancel: what its fp64 evaluation rounds
    if kind == fused.GAUSSIAN:
        vr = (do.base_dist.scale / d.base_dist.scale) ** 2
        t1 = ((do.base_dist.loc - d.base_dist.loc) / d.base_dist.scale) ** 2
        kl_terms = (0.5 * (vr + t1 + 1 + vr.log().abs())).sum(-1)
    else:
        fin = lambda t: torch.where(torch.isfinite(t), t.abs(), 0.0)  # noqa: E731
        kl_terms = (do.probs * (fin(do.logits) + fin(d.logits))).sum(-1)
    ratio_adv = torch.exp(lp - lp_old.double()) * adv_in.double()
    c = agent64.entropy_coef
    grads = torch.autograd.grad(gain, p)
    mag = lambda t: float(t.detach().abs().nan_to_num(0.0, 0.0, 0.0).mean())  # noqa: E731
    return (float(gain), float(kl_rows.mean()), float(ent.mean()),
            mag(ratio_adv) + c * mag(ent), mag(kl_terms), mag(ent), grads)


def run_stages(head, N, standardize, entropy_coef, monkeypatch, plant=True, zero_adv=False):
    import pfrl_b200
    from pfrl_b200.agents.trpo import (_distribution_params, _flatten_and_concat_variables,
                                       _hessian_vector_product)

    seed = N * 13 + len(head) + 2 * standardize + int(100 * entropy_coef)
    policy = make_policy(head, seed)
    pol64 = copy.deepcopy(policy).double().to(DEV)
    agent = pfrl_b200.agents.TRPO(policy, nn.Linear(OBS, 1), None, gpu=0, max_kl=0.01,
                                  entropy_coef=entropy_coef,
                                  standardize_advantages=standardize,
                                  conjugate_gradient_damping=0.1)
    agent64 = pfrl_b200.agents.TRPO(pol64, nn.Linear(OBS, 1), None, gpu=0, max_kl=0.01,
                                    entropy_coef=entropy_coef, conjugate_gradient_damping=0.1)
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(N, OBS, generator=g).to(DEV)
    with torch.no_grad():
        d = policy(s)
        a = d.sample()
        lp_old = d.log_prob(a).float()
    adv = torch.zeros(N, device=DEV) if zero_adv else torch.randn(N, generator=g).to(DEV)
    stats = torch.stack([adv.mean(), adv.std(unbiased=False)]) if standardize else None
    adv_in = (adv - stats[0]) / (stats[1] + 1e-8) if standardize else adv
    kind = agent._fused_kind(s)
    assert kind is not False
    P = sum(p.numel() for p in policy.parameters())
    vecs = [torch.randn(P, generator=torch.Generator().manual_seed(seed + i)).to(DEV)
            for i in range(3)]
    theta_old = _flatten_and_concat_variables([p.detach() for p in policy.parameters()])
    spy = _Spy(monkeypatch, agent, vecs)
    cand_out, gain_out, record = agent._policy_kernels(kind, s, a, lp_old, adv, stats)
    monkeypatch.undo()
    where = "%s N=%d std=%s c=%g" % (head, N, standardize, entropy_coef)
    s64 = s.double()
    params64 = list(pol64.parameters())

    # 1. the gain at theta_old, and its flat gradient J^T g
    dp, old = spy.gain_in
    g64 = fp64_objective(agent64, kind, dp, old, a, lp_old, adv_in)
    gain, _, ent, Sg, _, Se, gdp = g64
    check(where + ": gain", gain_out[0], gain, U * abs(gain) + 2.0 ** -36 * Sg)
    check(where + ": entropy", gain_out[2], ent, U * abs(ent) + 2.0 ** -36 * Se)
    assert float(gain_out[1]) == 0.0  # KL(old || old)
    D_ = raw_params(pol64, s64[:1]).shape[1]
    body = pol64.body if isinstance(pol64, _MaskedMLP) else pol64
    h2 = torch.tanh(body[0](s64)).pow(2)
    C = 2 * (N + OBS + H + 2 * D_ + 64) + 16 * float((h2 / (1 - h2)).max())
    # the fp64 gradient through the fp64 policy, seeded with the fp64 d gain / d params
    d64 = _distribution_params(pol64(s64))[1]
    with_grad = [i for i, x in enumerate(d64) if x.requires_grad]
    flat64 = _flatten_and_concat_variables(torch.autograd.grad(
        [d64[i] for i in with_grad], params64, [gdp[i] for i in with_grad]))
    # |g| in the raw parameters: the categorical's normalisation (I - 1 p^T) maps |g| to
    # at most |g| + p sum|g|
    if kind == fused.GAUSSIAN:
        gabs = torch.cat([gdp[0].abs(), (gdp[1].abs() if len(gdp) > 1 and 1 in with_grad
                                         else torch.zeros_like(gdp[0]))], 1)
    else:
        pr = D.Categorical(logits=dp[0].double()).probs
        gabs = gdp[0].abs() + pr * gdp[0].abs().sum(1, keepdim=True)

    # 2. the Fisher-vector product for three vectors, against the fp64 double-backward HVP
    dist = pol64(s64)
    with torch.no_grad():
        dist_old = pol64(s64)
    kl = torch.mean(D.kl_divergence(dist_old, dist))
    kl_grads = _flatten_and_concat_variables(
        torch.autograd.grad([kl], params64, create_graph=True))
    d_raw = raw_params(pol64, s64).detach()
    if kind == fused.GAUSSIAN:
        A_ = d_raw.shape[1] // 2
        sd = d_raw[:, A_:]
        mdiag = torch.cat([1 / sd ** 2, 2 / sd ** 2], 1) / N
        if head == "gauss_fixed":
            mdiag[:, A_:] = 0.0
        absM = lambda w: mdiag * w  # noqa: E731
    else:
        pr = torch.softmax(d_raw, 1)
        absM = lambda w: (pr * w + pr * (pr * w).sum(1, keepdim=True)) / N  # noqa: E731
    x, Ax, full, dId = spy.cg_step_io
    jt, jv = abs_jacobian_products(pol64, s64, [gabs], [v.double() for v in vecs])
    check(where + ": flat gain gradient", spy.b, flat64,
          C * U * jt[0] + U * flat64.abs() + 1e-300)
    jt_m, _ = abs_jacobian_products(pol64, s64, [absM(j) for j in jv], [])
    for i, v in enumerate(vecs):
        vd = v.double()
        want = _hessian_vector_product(kl_grads, params64, vd) + 0.1 * vd
        check(where + ": Fv %d" % i, spy.fvp_out[i], want,
              C * U * jt_m[i] + 2 * U * (want.abs() + 0.1 * vd.abs()) + 1e-300)

    # 3. dId and the full step, on the fused path's own x and F x
    check_cg_step(x, Ax, agent.max_kl, full, dId, where)

    # 4. every candidate's improvement and KL, on its fp32 distribution parameters
    n_cand = agent.line_search_max_backtrack + 1
    assert len(spy.cands) == n_cand
    vals = []
    for i, (cp, out) in enumerate(spy.cands):
        assert bits_equal(out, cand_out[i])
        gi, kli, _, Sgi, Skl, _, _ = fp64_objective(agent64, kind, cp, old, a, lp_old, adv_in)
        bg = U * abs(gi) + 2.0 ** -36 * Sgi
        bk = U * abs(kli) + 2.0 ** -36 * Skl
        check(where + ": candidate %d gain" % i, out[0], gi, bg)
        check(where + ": candidate %d KL" % i, out[1], kli, bk)
        # improvement = gain_i - gain_0: both bounds
        vals.append((gi - gain, kli, bg + U * abs(gain) + 2.0 ** -36 * Sg, bk))

    # 5. the decision, the record and the written parameters
    def decide(max_kl):
        """(fp64 winner, whether every candidate up to it clears its bound)."""
        for i, (imp, kli, bi, bk) in enumerate(vals):
            if not (math.isfinite(imp) and math.isfinite(kli)):
                continue
            clear = abs(imp) > bi and abs(kli - max_kl) > bk
            if imp >= 0 and kli <= max_kl:
                return i, clear
            if not clear:
                return None, False
        return -1, True

    theta, rec = spy.ls_out
    rec = rec.cpu().tolist()
    win = int(round(-math.log2(rec[1]))) if rec[2] == 1.0 else -1
    want, clear = decide(agent.max_kl)
    if clear:
        assert win == want, (where, win, want, vals)
    written = _flatten_and_concat_variables([p.detach() for p in policy.parameters()])
    assert bits_equal(written, theta)
    if win < 0:
        assert rec == [0.0, 0.0, 0.0] and bits_equal(theta, theta_old)
    else:
        assert rec[0] == float(cand_out[win, 1])
        want_theta = theta_old.cpu().numpy() + np.float32(2.0 ** -win) * full.cpu().numpy()
        assert bits_equal(theta, torch.from_numpy(want_theta))
    if plant and math.isfinite(vals[0][1]) and vals[0][0] > vals[0][2]:
        # candidate 0 two bounds either side of max_kl: accepted above, rejected below
        kl0, bk0 = vals[0][1], vals[0][3]
        for max_kl, accept in ((kl0 + 2 * bk0, True), (kl0 - 2 * bk0, False)):
            _, r = fused.line_search(cand_out, gain_out, max_kl, theta_old, full)
            got0 = float(r[1]) == 1.0
            assert got0 == accept == (decide(max_kl)[0] == 0), (where, max_kl, kl0)
    return agent, policy, pol64, (s, a, lp_old, adv, stats), record


@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("N", [1, 64, 257, 2048])
@pytest.mark.parametrize("standardize", [True, False])
@pytest.mark.parametrize("entropy_coef", [0.0, 0.01])
def test_fused_policy_update_stage_by_stage(head, N, standardize, entropy_coef, monkeypatch):
    run_stages(head, N, standardize, entropy_coef, monkeypatch)


@pytest.mark.parametrize("head", HEADS)
def test_zero_gradient_restores_theta_old_like_the_reference(head, monkeypatch):
    """Zero advantages, no entropy bonus, no standardisation: the gain's gradient b is 0,
    CG gives 0 / 0 = NaN, every candidate is NaN and the update restores theta_old bit for
    bit with step size 0, as the reference's formulation (here in fp64) does when
    torch.distributions does not validate its arguments (with validation on, the NaN
    candidate parameters make the policy's distribution raise instead)."""
    from pfrl_b200.agents.trpo import _flatten_and_concat_variables

    agent, policy, pol64, (s, a, lp_old, adv, _), record = run_stages(
        head, 64, False, 0.0, monkeypatch, plant=False, zero_adv=True)
    assert record.cpu().tolist() == [0.0, 0.0, 0.0]
    before = [p.detach().clone() for p in pol64.parameters()]
    import pfrl_b200

    agent64 = pfrl_b200.agents.TRPO(pol64, nn.Linear(OBS, 1), None, gpu=0, entropy_coef=0.0,
                                    standardize_advantages=False,
                                    conjugate_gradient_damping=0.1)
    with no_distribution_validation():  # as the fused path; validation rejects NaN params
        agent64._update_policy_torch(s.double(), a, lp_old.double(), adv.double())
    assert list(agent64.policy_step_size_record.host) == [0.0]
    for p, q in zip(before, pol64.parameters()):
        assert bits_equal(p, q)
    # the fp32 parameters are the fp64 ones, unchanged
    assert bits_equal(_flatten_and_concat_variables(list(policy.parameters())).double(),
                      _flatten_and_concat_variables(before))


# ------------------------------------------------------------- policies that are not fp32
@pytest.mark.parametrize("dtype", [torch.float64, torch.float16, torch.bfloat16],
                         ids=["fp64", "fp16", "bf16"])
@pytest.mark.parametrize("head", ["gauss_diagonal", "softmax18"])
def test_non_fp32_policy_takes_the_reference_formulation(dtype, head):
    """An fp64, fp16 or bf16 policy on CUDA gets the same update as use_fused=False."""
    import pfrl_b200

    results = []
    for use_fused in (True, False):
        policy = make_policy(head, 5).to(dtype)
        agent = pfrl_b200.agents.TRPO(policy, nn.Linear(OBS, 1), None, gpu=0)
        agent.use_fused = use_fused
        g = torch.Generator().manual_seed(6)
        s = torch.randn(300, OBS, generator=g).to(DEV, dtype)
        with torch.no_grad():
            d = agent.policy(s)
            a = d.sample() if head.startswith("softmax") else \
                (d.mean + torch.randn(d.mean.shape, generator=g).to(DEV, dtype))
            lp_old = d.log_prob(a)
        adv = torch.randn(300, generator=g).to(DEV, dtype)
        torch.manual_seed(0)
        agent._update_policy(s, a, lp_old, adv, torch.stack([adv.mean(), adv.std(unbiased=False)]))
        assert agent._line_search_log is None  # the fused path did not run
        results.append([p.detach().clone() for p in agent.policy.parameters()])
    for p, q in zip(*results):
        assert bits_equal(p, q)
