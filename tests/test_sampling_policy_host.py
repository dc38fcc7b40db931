"""CPU: the sampling policy's numpy restatement on hand-made rows, the new ABI symbols, and the refusals of the ABI and
of the Python entry points, which all happen before any CUDA call."""
import ctypes

import numpy as np
import pytest

from tests import sampling_policy_reference as R

INF = np.inf


def test_ties_at_the_kth_place_go_to_the_lower_index():
    o = np.array([1.0, 3.0, 3.0, 3.0, 0.0, -INF])
    assert list(R.ranking(o)) == [1, 2, 3, 0, 4]
    q, kept, _ = R.policy(o, 1.0, 2, 1.0)
    assert list(kept) == [1, 2]
    assert np.allclose(q, [0, 0.5, 0.5, 0, 0, 0])


def test_top_k_larger_than_the_finite_count_keeps_every_finite_entry():
    o = np.array([-INF, 1.0, 2.0, -INF])
    q, kept, _ = R.policy(o, 1.0, 5, 1.0)
    assert sorted(kept) == [1, 2]
    e = np.exp([1.0 - 2.0, 0.0])
    assert np.allclose(q[[1, 2]], e / e.sum()) and q[0] == q[3] == 0


def test_tiny_top_p_keeps_the_first_entry_of_the_ranking():
    o = np.array([0.5, 2.0, 2.0, 1.0])
    q, kept, _ = R.policy(o, 0.7, 0, 1e-6)
    assert list(kept) == [1] and q[1] == 1.0


def test_top_p_keeps_the_shortest_prefix_reaching_the_threshold():
    o = np.log(np.array([0.1, 0.4, 0.3, 0.2]))
    _, kept, margin = R.policy(o, 1.0, 0, 0.7)           # 0.4 + 0.3 = 0.7 reaches 0.7 of the total
    assert list(kept) == [1, 2] and margin < 1e-12
    _, kept, _ = R.policy(o, 1.0, 0, 0.71)
    assert list(kept) == [1, 2, 3]
    _, kept, _ = R.policy(o, 1.0, 3, 0.95)               # top-p over the top-k set: 0.95 of 0.9
    assert list(kept) == [1, 2, 3]


def test_temperature_zero_is_the_argmax_with_the_lowest_index():
    o = np.array([1.0, 4.0, -INF, 4.0])
    for k, p in ((0, 1.0), (3, 0.5)):
        q, kept, _ = R.policy(o, 0.0, k, p)
        assert list(kept) == [1] and q[1] == 1.0
    assert R.draw(R.policy(o, 0.0, 0, 1.0)[0], 0.999)[0] == 1


def test_temperature_flattens_and_sharpens_without_changing_the_ranking():
    o = np.array([0.0, 1.0, 2.0])
    hot, _, _ = R.policy(o, 4.0, 0, 1.0)
    cold, _, _ = R.policy(o, 0.25, 0, 1.0)
    assert hot[2] < np.exp(2) / np.exp(o).sum() < cold[2]
    assert list(R.ranking(o)) == [2, 1, 0]


def test_draw_is_the_index_order_inverse_cdf_and_skips_zero_weights():
    q = np.array([0.0, 0.25, 0.0, 0.75])
    assert R.draw(q, 0.0)[0] == 1 and R.draw(q, 0.2499)[0] == 1 and R.draw(q, 0.25)[0] == 3
    assert R.draw(q, 0.99999999)[0] == 3


def test_degenerate_rows():
    assert R.degenerate([-INF, -INF]) and R.degenerate([0.0, np.nan]) and R.degenerate([INF, 0.0])
    assert not R.degenerate([-INF, 0.0])


def test_model_probability_is_the_masked_softmax():
    o = np.array([0.0, np.log(3.0), -INF])
    assert abs(R.model_prob(o, 1) - 0.75) < 1e-15


def test_new_abi_symbols_are_exported():
    from graphinvent_b200 import _lib
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("gib_sampling_policy_set", "gib_sample_actions_policy", "gib_generation_sample_round_policy",
                 "gib_generation_sample_round_scaffold_policy", "gib_rl_sample_round_policy",
                 "gib_rl_sample_round_scaffold_policy"):
        assert hasattr(raw, name) and name in _lib.exported_symbols(), name
    assert ctypes.sizeof(_lib.SamplingPolicy) == 16


@pytest.mark.parametrize("t,k,p,word", [(-0.5, 0, 1.0, "temperature"), (float("inf"), 0, 1.0, "temperature"),
                                        (float("nan"), 0, 1.0, "temperature"), (1.0, -1, 1.0, "top_k"),
                                        (1.0, 0, 0.0, "top_p"), (1.0, 0, 1.5, "top_p"),
                                        (1.0, 0, float("nan"), "top_p")])
def test_abi_refuses_bad_policies_before_any_launch(t, k, p, word):
    from graphinvent_b200._lib import lib
    fake = ctypes.c_void_p(0x1000)            # never dereferenced: the refusal comes first
    assert lib.gib_sampling_policy_set(fake, t, k, p, None) == -1
    assert word in lib.gib_last_error().decode()


def test_abi_refuses_null_pointers():
    from graphinvent_b200._lib import lib
    fake = ctypes.c_void_p(0x1000)
    assert lib.gib_sampling_policy_set(None, 1.0, 0, 1.0, None) == -1
    assert "null" in lib.gib_last_error().decode()
    for args in ((None, 4, 9, fake, fake, fake, fake, None), (fake, 4, 9, None, fake, fake, fake, None),
                 (fake, 4, 9, fake, fake, None, fake, None), (fake, 4, 9, fake, None, fake, fake, fake),
                 (fake, 4, 0, fake, fake, fake, fake, None)):
        assert lib.gib_sample_actions_policy(*args, None) == -1
        assert "gib_sample_actions_policy" in lib.gib_last_error().decode()


@pytest.mark.parametrize("kw,word", [(dict(temperature=-1.0), "temperature"), (dict(temperature=float("nan")), "temperature"),
                                     (dict(temperature=1e39), "temperature"), (dict(top_k=-2), "top_k"),
                                     (dict(top_k=2.5), "top_k"), (dict(top_k=True), "top_k"),
                                     (dict(top_p=0.0), "top_p"), (dict(top_p=1.01), "top_p"),
                                     (dict(top_p=1e-50), "top_p")])
def test_python_refuses_bad_policies_naming_the_argument(kw, word):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGenerator, GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGenerator, GraphedGeneratorRL
    with pytest.raises(ValueError, match=word):
        Fn.sampling_policy(**kw)
    for cls in (GraphGenerator, GraphGeneratorRL, GraphedGenerator, GraphedGeneratorRL):
        with pytest.raises(ValueError, match=word):       # checked before the model or the device is touched
            cls(None, 4, **kw)


def test_python_policy_values_are_what_the_device_reads():
    from graphinvent_b200 import functional as Fn
    assert Fn.sampling_policy() == Fn.SAMPLING_OFF == (1.0, 0, 1.0)
    pol = Fn.sampling_policy(0.7, np.int64(10), 0.9)
    assert pol.top_k == 10 and isinstance(pol.top_k, int)
    assert pol.temperature == float(np.float32(0.7)) and pol.top_p == float(np.float32(0.9))
