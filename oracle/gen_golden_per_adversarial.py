"""Generate tests/golden/per_adversarial.npz from the REAL reference PrioritizedBuffer.

TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available:

    python oracle/gen_golden_per_adversarial.py

Drives pfrl/collections/prioritized.py (PrioritizedBuffer) on CPU with adversarial
priorities and chosen uniforms.  np.random.uniform is patched so that the reference
consumes u as 0.0 + root * u, exactly what numpy's uniform(0.0, root) computes from a
random_sample() of u.  The module-level _find is wrapped to record, for every draw, the
root it saw and the smallest |pos - left| along its own descent, relative to the root.

Scenarios: capacities 5, 1000 and 3000, filled partly or past capacity so that the
absolute pop counter sits at P - 1, P, P + 1 or 2P - 1 (mod 2P); priorities all equal,
powers of two, log-uniform over 1e-300..1e300, one dominant leaf among tiny ones,
subnormals, huge and tiny alternating; uniforms random, 0.0 and 1 - 2^-53, and
prefix / root of chosen leaves with their nextafter neighbours +-1..3.  A batch whose
descent ends on an empty slot makes the reference raise (AssertionError in
prioritized_sample, or ValueError in _find); that is recorded and ends the scenario.

The archive is written with fixed zip timestamps, so it regenerates byte-identically.
"""
import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "per_adversarial.npz")
FAMILIES = ("equal", "pow2", "loguniform", "dominant", "subnormal", "alternating")
TARGETS = ("partial", "P-1", "P", "P+1", "2P-1")
UKINDS = ("boundary", "ends", "random", "boundary")


def priorities(family, rng, n):
    if family == "equal":
        return [0.75] * n
    if family == "pow2":
        return [float(x) for x in np.ldexp(1.0, rng.randint(-60, 61, n))]
    if family == "loguniform":
        return [float(x) for x in 10.0 ** rng.uniform(-300, 300, n)]
    if family == "dominant":
        p = [1e-12] * n
        p[int(rng.randint(n))] = 1e6
        return p
    if family == "subnormal":
        return [float(k) * 5e-324 for k in rng.randint(1, 1 << 20, n)]
    return [1e300 if i % 2 == 0 else 1e-300 for i in range(n)]


def uniforms(kind, rng, n, live):
    if kind == "random":
        return [float(x) for x in rng.random_sample(n)]
    if kind == "ends":
        return [0.0 if i % 2 == 0 else 1.0 - 2.0 ** -53 for i in range(n)]
    # prefix / root in the reference's descent order (logical index order)
    pre = np.concatenate([[0.0], np.cumsum(live)[:-1]])
    root = float(np.sum(live))
    cand = pre[np.asarray(live) > 0] / root
    us = []
    for u0 in cand[rng.randint(len(cand), size=n // 7 + 1)]:
        us.append(u0)
        for step in (2.0, -1.0):
            v = u0
            for _ in range(3):
                v = np.nextafter(v, step)
                us.append(v)
    return [float(min(max(v, 0.0), 1.0 - 2.0 ** -53)) for v in us[:n]]


def main():
    import_reference()
    import pfrl.collections.prioritized as prio

    find0 = prio._find
    calls = []

    depth = [0]

    def find(ixl, ixr, node, pos):
        if depth[0]:  # _find recurses through the module global: only the top call is traced
            return find0(ixl, ixr, node, pos)
        root = node[2]
        margin = np.inf
        lo, hi, nd, p = ixl, ixr, node, pos
        while hi - lo > 1:
            left_node, right_node, _ = nd
            c = (lo + hi) // 2
            left = left_node[2] if left_node else 0.0
            margin = min(margin, abs(p - left) / root if root > 0 else np.inf)
            if p < left:
                hi, nd = c, left_node
            else:
                lo, nd, p = c, right_node, p - left
            if not nd and hi - lo > 1:
                break
        calls.append([root, margin, -1])
        depth[0] = 1
        try:
            calls[-1][2] = find0(ixl, ixr, node, pos)
        finally:
            depth[0] = 0
        return calls[-1][2]

    prio._find = find
    rng = np.random.RandomState(20261016)
    g = {k: [] for k in ("s_cap", "s_app_off", "b_scen", "b_u_off", "b_n", "b_raised",
                         "b_done", "b_redraw", "b_new_off", "b_total", "d_index", "d_prio",
                         "d_root", "d_margin", "app", "u", "new")}
    s = 0
    for cap in (5, 1000, 3000):
        P = 1
        while P < cap:
            P <<= 1
        for fi, fam in enumerate(FAMILIES):
            target = TARGETS[(fi + cap) % len(TARGETS)]
            total = {"partial": max(1, cap - cap // 3), "P-1": cap + P - 1, "P": cap + P,
                     "P+1": cap + P + 1, "2P-1": cap + 2 * P - 1}[target]
            buf = prio.PrioritizedBuffer(capacity=cap)
            app = priorities(fam, rng, total)
            g["s_cap"].append(cap)
            g["s_app_off"].append(len(g["app"]))
            g["app"].extend(app)
            for p in app:
                buf.append(None, p)
            live = list(app[-min(cap, total):])
            for bi, kind in enumerate(UKINDS):
                n = min(len(live), 64)
                u = uniforms(kind, rng, n, live)
                it = iter(u)
                np.random.uniform = lambda lo, hi: lo + (hi - lo) * next(it)  # noqa: E731
                g["b_scen"].append(s)
                g["b_u_off"].append(len(g["u"]))
                g["u"].extend(u)
                g["b_n"].append(n)
                g["b_total"].append(buf.priority_sums.sum())
                calls.clear()
                try:
                    ixs, vals = buf.priority_sums.prioritized_sample(n, remove=True)
                    raised, done = 0, n
                except (AssertionError, ValueError):
                    raised, done = 1, len(calls) - 1
                    cur = list(live)
                    ixs, vals = [], []
                    for root, margin, ix in calls[:done]:
                        ixs.append(ix)
                        vals.append(cur[ix])
                        cur[ix] = 0.0
                for k, (root, margin, _) in enumerate(calls):
                    g["d_index"].append(ixs[k] if k < done else calls[k][2])
                    g["d_prio"].append(vals[k] if k < done else np.nan)
                    g["d_root"].append(root)
                    g["d_margin"].append(margin)
                g["b_raised"].append(raised)
                g["b_done"].append(done)
                g["b_redraw"].append(int(len(set(ixs)) < len(ixs)))
                g["b_new_off"].append(len(g["new"]))
                if raised:
                    break
                new = priorities(FAMILIES[(fi + bi) % len(FAMILIES)], rng, n)
                g["new"].extend(new)
                buf.sampled_indices = ixs
                buf.flag_wait_priority = True
                buf.set_last_priority(new)
                for i, p in zip(ixs, new):
                    live[i] = p
            s += 1
    arrays = {k: np.asarray(v, dtype=np.float64 if k in ("b_total", "d_prio", "d_root",
                                                          "d_margin", "app", "u", "new")
                            else np.int64) for k, v in g.items()}
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with zipfile.ZipFile(OUT, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            bio = io.BytesIO()
            np.lib.format.write_array(bio, arrays[k], allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), bio.getvalue(),
                       compress_type=zipfile.ZIP_DEFLATED)
    print("numpy", np.__version__, "draws", len(g["d_index"]), "batches", len(g["b_n"]),
          "raised", sum(g["b_raised"]), "ties", int(np.sum(arrays["d_margin"] == 0)),
          "bytes", os.path.getsize(OUT))


if __name__ == "__main__":
    main()
