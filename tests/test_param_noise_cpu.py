"""DQN parameter-space noise without a GPU: the threshold deepq.learn hands to act, the float32 state machine the GPU
tests compare against, and the arguments that are refused."""
import numpy as np
import pytest

import _layer_norm_refs as L


@pytest.mark.parametrize("eps,nA", [(1.0, 2), (0.5, 4), (0.02, 6), (0.0, 3)])
def test_threshold_is_the_kl_of_eps_greedy(eps, nA):
    """deepq.py:274.  -log(1 - eps + eps / nA) is KL(greedy || eps-greedy): the greedy action keeps that probability."""
    from baselines_b200.deepq.deepq import param_noise_threshold
    got = param_noise_threshold(eps, nA)
    p = np.full(nA, eps / nA)
    p[0] += 1.0 - eps
    assert np.isclose(got, -np.log(p[0]), rtol=1e-12, atol=1e-15)
    assert got >= 0 and (got == 0) == (eps == 0.0)


def test_state_machine_sticky_values_and_order():
    s = L.ParamNoiseState()
    s.call(0.0, update_param_noise_threshold=-1)                       # negative: keep
    assert s.threshold == np.float32(0.05) and s.scale == np.float32(0.01) and s.eps == 0
    s.call(0.01, reset=True, update_param_noise_threshold=0.2, update_param_noise_scale=True, update_eps=0.3)
    assert s.reset_scale == np.float32(0.01)                            # the reset used the scale before the update
    assert s.scale == np.float32(np.float32(0.01) * np.float32(1.01)) and s.threshold == np.float32(0.2)
    assert s.eps == np.float32(0.3)
    s.call(0.5, update_param_noise_threshold=0.2, update_param_noise_scale=True)
    assert s.scale == np.float32(np.float32(np.float32(0.01) * np.float32(1.01)) / np.float32(1.01))
    s.call(0.0)                                                         # the default False == 0.0 replaces the threshold
    assert s.threshold == 0 and s.eps == np.float32(0.3)


def test_mean_kl_reference():
    rng = np.random.RandomState(0)
    q = rng.randn(7, 5)
    assert L.mean_kl(q, q) == 0.0 and L.mean_kl(q, q + 3.0) < 1e-15      # softmax is shift invariant
    r = rng.randn(7, 5)
    p, s = np.exp(q) / np.exp(q).sum(1, keepdims=True), np.exp(r) / np.exp(r).sum(1, keepdims=True)
    assert np.isclose(L.mean_kl(q, r), np.mean([sum(p[i, j] * np.log(p[i, j] / s[i, j]) for j in range(5))
                                                for i in range(7)]), rtol=1e-12)


def test_philox_normals_have_unit_moments():
    n = L.philox_normals(1234, 5, np.arange(40000))
    assert abs(n.mean()) < 0.02 and abs(n.std() - 1.0) < 0.02 and abs((n ** 3).mean()) < 0.05
    assert not np.array_equal(n, L.philox_normals(1234, 6, np.arange(40000)))


def test_custom_filter_is_refused():
    from baselines_b200.deepq.build_graph import build_train
    with pytest.raises(NotImplementedError, match="param_noise_filter_func"):
        build_train(num_actions=2, param_noise=True, param_noise_filter_func=lambda v: True)
