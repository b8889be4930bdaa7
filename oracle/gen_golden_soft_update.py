"""Generate tests/golden/soft_update.npz from the REAL reference soft_copy_param.

TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available:

    python oracle/gen_golden_soft_update.py

Runs pfrl/utils/copy_param.py:9-22 (soft_copy_param) on the CPU over the networks of
tests/soft_update_ref.py: Linear + BatchNorm1d MLPs in fp32, fp64, fp16 and bf16 (source
and target with different num_batches_tracked), a Linear tied under two names, a
transposed-view and a strided buffer, zero-size buffers and parameters, and fp32 / fp64 /
fp16 tensors seeded with NaN, +-inf, -0.0 and subnormals.  Each network gets the update
sequence TAUS; the target's state_dict is recorded before the first update and after
every one.  Keys: "<net>__init_target__<entry>", "<net>__init_source__<entry>",
"<net>__step<i>__<entry>"; bf16 entries are stored as their uint16 bit patterns.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.refimport import import_reference  # noqa: E402
from soft_update_ref import NETS, TAUS, make_pair, to_numpy  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "soft_update.npz")


def main():
    import_reference()
    from pfrl.utils.copy_param import soft_copy_param

    g = {"taus": np.array(TAUS, dtype=np.float64)}
    for name in NETS:
        target, source = make_pair(name)
        for tag, net in (("init_target", target), ("init_source", source)):
            for k, v in net.state_dict().items():
                g["%s__%s__%s" % (name, tag, k)] = to_numpy(v)
        for i, tau in enumerate(TAUS):
            soft_copy_param(target, source, tau)
            for k, v in target.state_dict().items():
                g["%s__step%d__%s" % (name, i, k)] = to_numpy(v)
    np.savez_compressed(OUT, **g)
    print("wrote %s: %d arrays, %d bytes" % (OUT, len(g), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
