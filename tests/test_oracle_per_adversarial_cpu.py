"""CPU: oracle/per_oracle.c against the real reference PrioritizedBuffer on adversarial trees
(tests/golden/per_adversarial.npz, written by oracle/gen_golden_per_adversarial.py).

Every draw's index and priority and every batch's total are bit-identical, as long as the
oracle's descents land on live leaves.  When pos = root * u rounds up to the whole live mass
(u = 1 - 2^-53, subnormal roots), the reference's descent ends on its newest leaf or raises
(an empty slot: AssertionError / ValueError), while the dense heap ends on an empty slot past
the live window (DESIGN §7a); the test checks that this is the only divergence and then ends
the scenario.  The fixture must keep its edge cases among the compared draws: exact ties
(pos == left at some level) and draws within v6's margin EPS = (n + 64) * 2^-46 * root.
"""
import os

import numpy as np

from oracle.replay import OraclePrioritizedBuffer

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "per_adversarial.npz")


def _draw_offsets(g):
    # draws recorded per batch: n, or done + 1 when the reference raised
    per = np.where(g["b_raised"] == 1, g["b_done"] + 1, g["b_n"])
    return np.concatenate([[0], np.cumsum(per)])


def test_oracle_is_bit_identical_to_reference_on_adversarial_trees():
    g = np.load(GOLDEN)
    off = _draw_offsets(g)
    app_end = np.concatenate([g["s_app_off"][1:], [len(g["app"])]])
    margins, sizes, stops = [], [], 0
    for s, cap in enumerate(g["s_cap"].tolist()):
        ora = OraclePrioritizedBuffer(cap)
        app = np.ascontiguousarray(g["app"][g["s_app_off"][s]:app_end[s]])
        for p in app.tolist():
            ora.append(None, p)
        for b in np.flatnonzero(g["b_scen"] == s).tolist():
            n = int(g["b_n"][b])
            u = np.ascontiguousarray(g["u"][g["b_u_off"][b]:g["b_u_off"][b] + n])
            live = int(ora._L.ora_per_live_prefix(ora._h, n, u.ctypes.data))
            idx, pri, tot, _ = ora.sample_indices(n, u)
            assert tot == g["b_total"][b], (s, b)
            d0 = off[b]
            done = int(g["b_done"][b])
            k = min(live, done)
            assert idx[:k].tolist() == g["d_index"][d0:d0 + k].tolist(), (s, b)
            assert pri[:k].tobytes() == g["d_prio"][d0:d0 + k].tobytes(), (s, b)
            margins.append(g["d_margin"][d0:d0 + k])
            sizes.append(np.full(k, n))
            if live < n or g["b_raised"][b]:
                # pos rounded up to the live mass: the oracle (and the device) land past the
                # live window, where the reference raises or takes its newest leaf
                assert live < n and idx[live] >= len(ora), (s, b)
                if g["b_raised"][b]:
                    assert live == done, (s, b, live, done)
                else:
                    assert g["d_index"][d0 + live] == len(ora) - 1, (s, b)
                stops += 1
                break
            ora.set_last_priority(g["new"][g["b_new_off"][b]:g["b_new_off"][b] + n])
    m = np.concatenate(margins)
    ties = int(np.sum(m == 0.0))
    within = int(np.sum(m < (np.concatenate(sizes) + 64) * 2.0 ** -46))
    print("compared draws %d, exact ties %d, within v6 EPS %d, scenarios stopped past the live "
          "window %d" % (len(m), ties, within, stops))
    assert ties > 0 and within > ties, (ties, within)
    assert stops > 0
