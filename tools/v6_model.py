"""CPU model of the v6 exact sampler's decision logic (tools, not product).

The main warp of k_sample_exact_v6 decides every draw on an APPROXIMATE copy A of the
top of the sum tree (updated by plain subtractions, all levels at once) and on the exact
bottom levels, and accepts a decision only when it is farther than EPS from every
boundary it crosses; otherwise the draw falls back to the reference's exact sequential
arithmetic.  This model checks, on adversarial trees, that the accepted decisions always
equal the exact chain's, and counts the fallbacks.
"""
import sys
from fractions import Fraction

import numpy as np


def build(leaves):
    n = len(leaves)
    h = np.zeros(2 * n)
    h[n:] = leaves
    for i in range(n - 1, 0, -1):
        h[i] = h[2 * i] + h[2 * i + 1]
    return h


def exact_draw(h, n, u, older=2):
    """reference arithmetic (collections/prioritized.py:245-258, 294-312)"""
    pos = h[1] * u
    node = older
    if not (pos < h[older]):
        pos = pos - h[older]
        node = older ^ 1
    while node < n:
        left = h[2 * node]
        if pos < left:
            node = 2 * node
        else:
            pos = pos - left
            node = 2 * node + 1
    return node


def zero_and_reduce(h, node):
    h[node] = 0.0
    p = node >> 1
    while p >= 1:
        h[p] = h[2 * p] + h[2 * p + 1]
        p >>= 1


WIN = 32  # leaves in the scout's window (one per lane)


def fma_sub(a, b, c):
    """a * b - c with one rounding (the DFMA nvcc contracts the kernel's expression to)"""
    return float(Fraction(a) * Fraction(b) - Fraction(c))


def warp_scan(p):
    """inclusive Hillis-Steele scan in the kernel's order (__shfl_up_sync by 1, 2, 4, 8, 16)"""
    incl = np.array(p, dtype=np.float64)
    o = 1
    while o < len(incl):
        nxt = incl.copy()
        nxt[o:] = incl[o:] + incl[:-o]
        incl = nxt
        o <<= 1
    return incl


def leaf_window(E, node, D, x, shift=0):
    """What a scout lays down for the staged subtree below heap node `node`: descend it at
    the predicted position x to a leaf, take the WIN leaves centred on it (clamped to the
    subtree; `shift` moves the window to model a bad prediction), and return the lower
    bound of every window leaf inside the node's interval, the window's end and its first
    leaf (relative to the subtree's first leaf)."""
    nleaf = 1 << D
    r = 1                            # relative heap index: node << j + r - 2^j at depth j
    for j in range(D):
        left = E[2 * ((node << j) + r - (1 << j))]
        right = not (x < left)
        x = x - left if right else x
        r = 2 * r + int(right)
    f = min(max(r - nleaf - WIN // 2 + shift, 0), nleaf - WIN)
    leaf0 = (node << D) + f
    base = 0.0  # left siblings on the path to the first leaf, top-down
    for j in range(D - 1, -1, -1):
        if (f >> j) & 1:
            base += E[(leaf0 >> j) - 1]
    p = E[leaf0:leaf0 + WIN]
    incl = warp_scan(p)
    lo = np.empty(WIN)
    lo[0] = base
    lo[1:] = base + incl[:-1]
    return lo, base + incl[-1], f


def run(leaves, us, T, eps_rel=None, older=2, mispredict=0.0, rng=None, prefetch=False,
        stats=None):
    """Prefix-table formulation of the kernel: M / P_lo / P_hi over the level-(T-1)
    nodes in descent order (older half first), the scout's leaf window under the
    predicted node; a draw is accepted only when pos is farther than EPS from both ends
    of the node's interval and of the leaf's interval.  eps_rel=None is the kernel's
    EPS = (n + 64) 2^-46 root for a launch of n = len(us) draws.

    prefetch=True models the main warp's pipeline: a draw's table entries are read before
    the previous draw's update is stored, and that one update is applied in registers
    (the prefix loses its priority when the previous node comes first in descent order; a
    draw at the previous draw's node is a conflict and takes the exact path).  The scout's
    window is then laid down from a staged copy of the exact tree that still lacks the
    previous draw, as a copy taken before that draw was applied does in the kernel: a
    decision at that node on that window can pick another leaf than the exact chain, which
    is what the conflict rule prevents.  stats, a dict, receives counts of the draws decided
    on corrected entries."""
    n = len(leaves)
    L = n.bit_length() - 1          # leaves at level L
    E = build(leaves)
    Ex = E.copy()                   # pure exact sampler for comparison
    ntop = 1 << (T - 1)             # nodes at level T-1
    flip = 0 if older == 2 else ntop // 2
    blk = max(1, int(np.sqrt(ntop)))
    while ntop % blk:
        blk -= 1
    M = np.array([E[ntop + (o ^ flip)] for o in range(ntop)])
    P_lo = np.zeros(ntop)
    P_hi = np.zeros(ntop // blk)
    run_hi = 0.0
    for b in range(ntop // blk):
        P_hi[b] = run_hi
        r = 0.0
        for i in range(blk):
            P_lo[b * blk + i] = r
            r += M[b * blk + i]
        run_hi += r
    def apply_update(od, prio):
        """approximate update: everything after the drawn node"""
        M[od] -= prio
        bb = od // blk
        P_lo[od + 1:(bb + 1) * blk] -= prio
        P_hi[bb + 1:] -= prio

    rootA = E[1]
    if eps_rel is None:
        eps_rel = (len(us) + 64) * 2.0 ** -46
    eps = eps_rel * E[1]
    D = L - (T - 1)
    assert D >= 5, "the window holds 32 leaves: at least 5 levels below the table level"
    fallbacks = 0
    out = []
    pending = None                  # (node, priority) of the draw whose update is not stored
    E_staged = E.copy()             # the exact tree without the pending draw (prefetch=True)
    if stats is not None:
        stats.update(before=0, after=0, same=0, accepted_before=0, accepted_after=0)
    for u in us:
        want = exact_draw(Ex, n, u, older)
        # ---- scout: predicted node and leaf from the tables (optionally perturbed)
        pos = rootA * u
        b = max(0, int(np.searchsorted(P_hi, pos, side="right")) - 1)
        w = max(0, int(np.searchsorted(P_lo[b * blk:(b + 1) * blk], pos - P_hi[b], side="right")) - 1)
        o = b * blk + w
        x = (pos - P_hi[b]) - P_lo[o]
        shift = 0
        if rng is not None and rng.rand() < mispredict:
            o = min(ntop - 1, max(0, o + rng.randint(-1, 2)))
        if rng is not None and rng.rand() < mispredict:
            shift = int(rng.randint(-40, 41))
        node = ntop + (o ^ flip)
        lo, end, f = leaf_window(E_staged if prefetch else E, node, D, x, shift)
        # ---- main: one vote against the window
        pre = P_hi[o // blk] + P_lo[o]
        mass = M[o]
        conflict = False
        side = None
        if pending is not None:     # the entries were read before the pending update
            op, pp = pending
            if op < o:
                pre -= pp
            conflict = op == o
            side = "before" if op < o else "same" if op == o else "after"
            apply_update(op, pp)
            pending = None
        pos12 = fma_sub(rootA, u, pre)
        leaf = None
        if not conflict and eps < pos12 < mass - eps:
            c = int(np.count_nonzero(pos12 >= lo)) - 1
            hi = end if c == WIN - 1 else lo[min(c + 1, WIN - 1)]
            if c >= 0 and pos12 - lo[c] > eps and hi - pos12 > eps:
                leaf = (node << D) + f + c
        if stats is not None and side is not None:
            stats[side] += 1
            if leaf is not None and side != "same":
                stats["accepted_" + side] += 1
        if leaf is None:
            fallbacks += 1
            leaf = exact_draw(E, n, u, older)
        assert leaf == want, ("decision differs from the exact chain", leaf, want, u)
        prio = E[leaf]
        out.append(leaf)
        if prefetch:
            E_staged = E.copy()
        zero_and_reduce(E, leaf)      # exact ascent (ascent warp)
        zero_and_reduce(Ex, leaf)
        od = ((leaf >> D) - ntop) ^ flip
        if prefetch:
            pending = (od, prio)
        else:
            apply_update(od, prio)
        rootA = rootA - prio
    if pending is not None:
        apply_update(*pending)
    assert np.array_equal(E, Ex)
    return out, fallbacks


def families(rng, n=1 << 12):
    """adversarial leaf sets: (name, leaves)"""
    sp = np.zeros(n)
    sp[rng.randint(0, n, 300)] = rng.rand(300)
    return [
        ("uniform random", rng.rand(n) + 0.01),
        ("all equal (ties on power-of-two sums)", np.ones(n)),
        ("huge dynamic range", np.exp(rng.randn(n) * 12)),
        ("sparse (mostly empty slots)", sp),
        ("tiny among big", np.where(rng.rand(n) < 0.5, 1e-30, 1.0)),
        ("1e-30 .. 1e+30", 10.0 ** rng.uniform(-30, 30, n)),
    ]


def draws(rng, leaves, k=256):
    """u for one launch, with u = 0, u just below 1 and u on node and leaf boundaries of
    equal trees"""
    k = min(k, int((leaves > 0).sum()))
    us = rng.random_sample(k)
    us[::17] = 0.0
    us[5::31] = np.nextafter(1.0, 0.0)
    us[3::13] = np.round(us[3::13] * 64) / 64
    us[7::11] = np.round(us[7::11] * len(leaves)) / len(leaves)
    return us


def main():
    rng = np.random.RandomState(0)
    total_fb = total = 0
    for name, leaves in families(rng):
        for T in (4, 7, 8):                 # 9, 6 and 5 levels below the table level
            for eps_rel in (None, 2.0 ** -20, 0.5):
                us = draws(rng, leaves)
                _, fb = run(leaves, us, T, eps_rel, older=2 + (T & 1), mispredict=0.05, rng=rng)
                total_fb += fb if eps_rel is None else 0
                total += len(us) if eps_rel is None else 0
                print("%-40s T=%d eps=%-8s draws=%d fallbacks=%d" % (
                    name, T, "kernel" if eps_rel is None else "2^%d" % np.log2(eps_rel),
                    len(us), fb))
    print("fallback rate at the kernel's EPS: %d / %d" % (total_fb, total))


if __name__ == "__main__":
    sys.exit(main())
