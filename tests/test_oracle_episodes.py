"""CPU: the oracle's multi-episode evaluations (obj.py:54-63, ``eps_per_policy``) and BatchedRollout's ``episodes``
argument."""
import numpy as np
import pytest

from oracle import es_oracle as orc

OBS, ACT, HID, T = 5, 3, (8, 8), 13          # T * ACT odd: the gaussian cache crosses episodes and evaluations


def _problem(seed=3):
    dims = orc.layer_dims(OBS, HID, ACT)
    P = orc.n_params(dims)
    rs = np.random.RandomState(seed)
    table = rs.randn(P + 5000).astype(np.float32)
    theta = (rs.randn(P) * 0.3).astype(np.float32)
    return dims, table, theta, orc.SyntheticEnvSpec(OBS, ACT, T)


def _streams(seeds):
    out = [np.random.RandomState(s) for s in seeds]
    out[0].randn(1)                                              # start with a cached gaussian
    return out


def _state(rs):
    st = rs.get_state()
    return st[1].copy(), st[2], st[3], st[4]


def _same_states(a, b):
    for x, y in zip(a, b):
        sx, sy = _state(x), _state(y)
        assert np.array_equal(sx[0], sy[0]) and sx[1:] == sy[1:]


def _test_params(episodes, ac_std, seeds=(21, 22), n=3, **kw):
    """es_test_params with ``episodes`` episodes per evaluation; None leaves the argument at its default."""
    dims, table, theta, env = _problem()
    streams = _streams(seeds)
    args = (table, theta, 0.05, dims, env, [None] * len(seeds), n, np.zeros(OBS), np.ones(OBS), 5.0, T)
    kw = dict(coins_per_eval=1, save_obs_chance=0.5, rank_states=streams, ac_std=ac_std, **kw)
    if episodes is not None:
        kw['episodes'] = episodes
    return orc.es_test_params(*args, **kw), streams


@pytest.mark.parametrize('ac_std', [0.0, 0.01])
def test_one_episode_is_the_oracle(ac_std):
    """``episodes=1`` is the single-episode path: values and stream state identical."""
    (pos, neg, inds, steps, ob), sa = _test_params(1, ac_std)
    (pos0, neg0, inds0, steps0, ob0), sb = _test_params(None, ac_std)
    assert np.array_equal(pos, pos0) and np.array_equal(neg, neg0) and np.array_equal(inds, inds0) and steps == steps0
    assert np.array_equal(ob.sum, ob0.sum) and np.array_equal(ob.sumsq, ob0.sumsq) and ob.count == ob0.count
    _same_states(sa, sb)


def test_one_episode_generation_and_step_are_the_oracle():
    dims, table, theta, env = _problem()
    P = len(theta)
    res = []
    for episodes in ({'episodes': 1}, {}):
        flat, opt, streams = theta.copy(), orc.AdamOracle(P, 0.01), _streams((5, 6))
        args = (table, flat, opt, 0.05, dims, env, streams, 2, np.zeros(OBS), np.ones(OBS), 5.0, T, 100, 0.005)
        out = orc.es_step(*args, coins_per_eval=1, save_obs_chance=0.5, ac_std=0.01, **episodes)
        res.append((out, flat, streams))
    (a, fa, sa), (b, fb, sb) = res
    assert np.array_equal(fa, fb) and a['noiseless'] == b['noiseless']
    for k in ('pos', 'neg', 'inds', 'weights'):
        assert np.array_equal(a[k], b[k])
    _same_states(sa, sb)


@pytest.mark.parametrize('episodes', [2, 3, 7])
def test_noiseless_episodes_change_nothing(episodes):
    """Without action noise the E episodes are identical: E copies of a float32 value sum exactly in float64 (E < 2^29) and
    (E r) / E == r, so fitness, indices, statistics and the stream are those of one episode, bit for bit."""
    (pos, neg, inds, steps, ob), sa = _test_params(episodes, 0.0)
    (pos1, neg1, inds1, steps1, ob1), sb = _test_params(1, 0.0)
    assert np.array_equal(pos, pos1) and np.array_equal(neg, neg1) and np.array_equal(inds, inds1) and steps == steps1
    assert np.array_equal(ob.sum, ob1.sum) and ob.count == ob1.count
    _same_states(sa, sb)


def test_noiseless_episode_mean_is_exact():
    """The arithmetic fact the noiseless case rests on, over many float32 values and episode counts."""
    r = np.random.RandomState(0).randn(2000).astype(np.float32) * np.float32(1e3)
    for e in (2, 3, 5, 7, 10, 1000, 123457):
        acc = np.zeros(len(r))
        for _ in range(min(e, 12)):
            acc += r.astype(np.float64)
        if e <= 12:
            assert np.array_equal(acc / e, r.astype(np.float64))
        assert np.array_equal((r.astype(np.float64) * e) / e, r.astype(np.float64))


@pytest.mark.parametrize('episodes', [2, 3])
def test_noisy_episodes_match_obj_py(episodes):
    """Against a literal transcription of obj.py:54-63's r_fn inside es.test_params (es.py:66-72): per pair the index, then
    per evaluation the coin and E episodes, each drawing T x rs.randn(act) from the rank's stream."""
    dims, table, theta, env = _problem()
    seeds, n, ac_std, std, chance = (21, 22), 3, 0.01, 0.05, 0.5
    (pos, neg, inds, _, ob), streams = _test_params(episodes, ac_std, seeds, n)
    ref_streams = _streams(seeds)
    fits, ref_inds, saved = [], [], 0
    for rs in ref_streams:
        for _ in range(n):
            idx = int(rs.randint(0, len(table) - len(theta)))
            ref_inds.append(idx)
            noise = table[idx:idx + len(theta)]
            for sign in (1, -1):
                save_obs = rs.random() < chance
                layers = orc.unflatten(orc.pheno_params(theta, std, noise if sign > 0 else -noise), dims)
                rews = np.zeros(T)
                for _ in range(max(1, episodes)):
                    rew, behv, obs, steps = orc.run_model(env, layers, np.zeros(OBS), np.ones(OBS), 5.0, T, True, ac_std, rs)
                    rews[:len(rew)] += np.array(rew)
                rews /= max(1, episodes)
                fits.append(sum(rews.tolist()))
                saved += int(save_obs)
    fits = np.array(fits).reshape(-1, 2)
    assert np.array_equal(pos[:, 0], fits[:, 0]) and np.array_equal(neg[:, 0], fits[:, 1])
    assert np.array_equal(inds, np.array(ref_inds, dtype=np.float64))
    assert ob.count == saved * T
    _same_states(streams, ref_streams)
    # and the episodes do matter when the actions are noisy
    (pos1, _, _, _, _), _ = _test_params(1, ac_std, seeds, n)
    assert not np.array_equal(pos, pos1)


def test_batched_rollout_episodes_argument():
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
    env = SyntheticEnv(OBS, ACT, T)
    assert BatchedRollout(env, T).episodes == 1
    assert BatchedRollout(env, T, episodes=0).episodes == 1                  # max(1, eps_per_policy), obj.py:57
    assert BatchedRollout(env, T, episodes=10).episodes == 10
    assert BatchedRollout(env, T, episodes=np.int64(3)).episodes == 3
    for bad in (2.0, 2.5, '3', True, None):
        with pytest.raises(TypeError):
            BatchedRollout(env, T, episodes=bad)
    with pytest.raises(ValueError):
        BatchedRollout(env, T, episodes=-1)
    archive = np.zeros((4, 2))
    assert BatchedRollout(env, T, archive=archive, episodes=1).episodes == 1
    with pytest.raises(ValueError):
        BatchedRollout(env, T, archive=archive, episodes=2)
