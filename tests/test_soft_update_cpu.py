"""Soft target updates on the CPU against the reference's own soft_copy_param
(pfrl/utils/copy_param.py:9-22), recorded in tests/golden/soft_update.npz by
oracle/gen_golden_soft_update.py: the line-for-line restatement in
tests/soft_update_ref.py and pfrl_b200.utils.copy_param.soft_copy_param must both
reproduce every recorded target state bit for bit (NaN payloads and signed zeros
included), over fp32 / fp64 / fp16 / bf16 nets, BatchNorm integer buffers, tied,
non-contiguous and zero-size entries and special values."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from soft_update_ref import (NETS, TAUS, array_bits, bits, from_numpy, make_pair,  # noqa: E402
                             reference_soft_copy)

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "soft_update.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


def _load(net, golden, prefix):
    with torch.no_grad():
        for k, v in net.state_dict().items():
            v.copy_(from_numpy(golden[prefix + k], v.dtype))


def _assert_state(net, golden, prefix, what):
    for k, v in net.state_dict().items():
        want = golden[prefix + k]
        assert tuple(v.shape) == want.shape, (what, k)
        np.testing.assert_array_equal(bits(v), array_bits(want, v), err_msg="%s %s" % (what, k))


def _soft_copy_param(target, source, tau):
    from pfrl_b200.utils.copy_param import soft_copy_param

    soft_copy_param(target, source, tau)


def test_fixture_covers_the_cases(golden):
    np.testing.assert_array_equal(golden["taus"], np.array(TAUS))
    assert golden["mlp_bn_fp32__init_target__1.num_batches_tracked"] != \
        golden["mlp_bn_fp32__init_source__1.num_batches_tracked"]
    s32 = golden["special_values__init_target__s32"]
    assert np.isnan(s32).any() and np.isinf(s32).any() and (np.signbit(s32) & (s32 == 0)).any()
    assert ((s32 != 0) & (np.abs(s32) < np.finfo(np.float32).tiny)).any()
    s16 = golden["special_values__init_source__s16"]
    assert ((s16 != 0) & (np.abs(s16) < np.finfo(np.float16).tiny)).any()
    assert golden["zero_size__step0__empty_2d"].shape == (3, 0)


@pytest.mark.parametrize("impl", [reference_soft_copy, _soft_copy_param],
                         ids=["restatement", "soft_copy_param"])
@pytest.mark.parametrize("name", NETS)
def test_soft_update_matches_reference_fixture(golden, name, impl):
    target, source = make_pair(name)
    _load(target, golden, "%s__init_target__" % name)
    _load(source, golden, "%s__init_source__" % name)
    for i, tau in enumerate(TAUS):
        impl(target, source, tau)
        _assert_state(target, golden, "%s__step%d__" % (name, i), (name, tau))
        # the source is only read
        _assert_state(source, golden, "%s__init_source__" % name, (name, tau, "source"))


def test_integer_and_bf16_entries_are_left_alone(golden):
    """What the fixture pins, spelled out: the reference rebinds non-averaged entries
    in a dict copy, so neither num_batches_tracked nor a bf16 tensor of the target
    moves."""
    from pfrl_b200.utils.copy_param import soft_copy_param

    target, source = make_pair("mlp_bn_bf16")
    before = {k: v.clone() for k, v in target.state_dict().items()}
    soft_copy_param(target, source, 0.37)
    for k, v in target.state_dict().items():
        assert torch.equal(v, before[k]), k
    assert target[1].num_batches_tracked != source[1].num_batches_tracked


def test_tied_parameter_is_averaged_twice():
    from pfrl_b200.utils.copy_param import soft_copy_param

    target, source = make_pair("tied")
    tau = 0.37
    d = target.first.weight.detach().clone()
    s = source.first.weight.detach()
    once = d * (1 - tau) + tau * s
    soft_copy_param(target, source, tau)
    assert torch.equal(target.first.weight, once * (1 - tau) + tau * s)
