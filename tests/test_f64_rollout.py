"""The float64 rollout reference (tests/f64_rollout.py) against the CPU oracle before anything is judged by it: same
fitness to float32 level, same final positions, for 1-5 hidden layers, one action, widths that are not multiples of 4,
with and without action noise and with 1 or 3 episodes."""
import os
import sys

import numpy as np
import pytest

from oracle import es_oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import f64_rollout as f64  # noqa: E402


class _Replay:
    """Stands in for the RandomState that run_model draws rs.randn(act) from: replays a fixed array, row by row."""

    def __init__(self, a):
        self.a, self.i = a.astype(np.float64), 0

    def randn(self, n):
        self.i += 1
        return self.a[self.i - 1]


@pytest.mark.parametrize('obs,hidden,act,T,E,noisy', [
    (5, (8,), 1, 7, 1, False),
    (15, (33, 6), 3, 40, 1, True),
    (9, (7, 13, 5), 4, 25, 3, True),
    (26, (21, 10, 17, 3), 6, 19, 1, False),
    (7, (11, 9, 6, 14, 5), 2, 30, 3, True),
    (13, (30, 30), 1, 33, 3, True),
])
def test_f64_reference_matches_the_oracle(obs, hidden, act, T, E, noisy):
    rs = np.random.RandomState(obs * 100 + T)
    sizes = [obs] + list(hidden) + [act]
    dims = orc.layer_dims(obs, hidden, act)
    P = orc.n_params(dims)
    assert f64.n_params(sizes) == P
    L = P + 5000
    table, theta = rs.randn(L).astype(np.float32), (rs.randn(P) * 0.3).astype(np.float32)
    n = 3
    idx = rs.randint(0, L - P, size=n)
    env = orc.SyntheticEnvSpec(obs, act, T)
    mean, std = rs.randn(obs) * 0.1, 0.5 + rs.rand(obs)
    obsn = orc.normalise_obs(env.obs_stream[:T], mean, std, 5.0)
    noise = (rs.randn(n, 2, E, T, act) * 0.05).astype(np.float32) if noisy else None
    sigma = 0.05
    fit, behv, mass, mag = f64.rollout_f64(table, idx, theta, sigma, sizes, obsn, env.rew_vec, env.pos_scale, noise,
                                           E if noisy else 1)
    for k in range(n):
        eps = orc.table_get(table, int(idx[k]), P)
        for s, nz in ((0, eps), (1, -eps)):
            layers = orc.unflatten(orc.pheno_params(theta, sigma, nz), dims)
            if noisy:
                rews, bb, _, _ = orc.run_model(env, layers, mean, std, 5.0, T, ac_std=1.0,
                                               rs=_Replay(noise[k, s].reshape(E * T, act)), episodes=E)
            else:
                rews, bb, _, _ = orc.run_model(env, layers, mean, std, 5.0, T)
            ref = orc.reward_result(rews)[0]
            # the oracle rounds weights, activations, actions and rewards to float32: ~1e-7 of the reward mass
            assert abs(fit[s, k] - ref) <= 2e-6 * mass[s, k], (k, s, fit[s, k], ref)
            assert mass[s, k] >= np.abs(rews).sum() * (1 - 1e-5)
            # float32 positions: the reference's position magnitude bounds their rounding, plus the float32 actions' error
            assert np.all(np.abs(behv[s, k] - bb[-3:]) <= 2 ** -24 * mag[s, k] + 1e-6 * env.pos_scale * T), (behv[s, k], bb[-3:])


def test_f64_reference_layout_and_noise_sign():
    """The flat layout is the state dict's (weight[out, in] row-major, then bias) and +-eps rows differ; sigma is taken as
    the float32 the kernels receive."""
    sizes = [3, 2, 1]
    assert f64.layer_slices(sizes) == [(0, 6, 3, 2), (8, 10, 2, 1)]
    theta = np.zeros(11, dtype=np.float32)
    table = np.arange(20, dtype=np.float32)
    w = f64.perturbed(table, 4, theta, 0.1, -1.0)
    assert np.array_equal(w, -float(np.float32(0.1)) * np.arange(4, 15, dtype=np.float64))
    obsn = np.ones((2, 3), dtype=np.float32)
    rew = np.ones((2, 1), dtype=np.float32)
    fit, behv, mass, _ = f64.rollout_f64(table, [4], theta, 0.1, sizes, obsn, rew, 0.5)
    for row, sg in ((0, 1.0), (1, -1.0)):
        e = sg * float(np.float32(0.1)) * np.arange(4, 15, dtype=np.float64)
        h = np.tanh(e[:6].reshape(2, 3) @ np.ones(3) + e[6:8])
        a = np.tanh(e[8:10] @ h + e[10])
        assert np.isclose(fit[row, 0], 2 * a, rtol=1e-15) and np.allclose(behv[row, 0], 0.5 * 2 * a, rtol=1e-15)
        assert np.isclose(mass[row, 0], abs(fit[row, 0]), rtol=1e-15)
