"""CPU (no GPU): episodes that end early on the closed-loop env (ClosedLoopEnv(fall_height=h)).

* the done rule: float32 |z| after the step's position update against float32 h, NaN falls, T still ends the episode;
* run_model's python loop on a terminating env against a restatement from the oracle's env and forward: rewards, t_d, the
  padded behaviour and the observation rows;
* obj.py's E-episode fold (BatchedRollout's python route) with a last episode shorter than an earlier one;
* the float64 truth (tests/closed_f64.py): a fall height nothing reaches is no fall height, for the truth and every modelled
  bug, and a NaN position ends an episode only when there is a fall height;
* argument validation, and the new entry points' declarations and bindings (the cluster kernel's compilation for sm_90a is
  checked in test_host_ptxas_closed_wide.py)."""
import os
import re
import sys
from typing import Optional

import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closed_f64 as cf  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def run_model_loop(env, model_fn, max_steps: int, rs: Optional[np.random.RandomState] = None, ac_std: float = 0.0):
    """run_model's python loop (gym_runner.py:33-67) restated on a ClosedLoopEnv-like ``env`` with the float32 forward
    ``model_fn(ob) -> action``: every step adds ``rs.randn(act) * ac_std`` when given, steps the env, records the reward,
    the observation and the position, and breaks on done; the behaviour is padded with the last position.  Returns (rews,
    behv, obs [steps][obs], step)."""
    behv, rews, obs = [], [], []
    ob = env.reset()
    step = 0
    for step in range(max_steps):
        a = np.asarray(model_fn(ob), dtype=F32)
        if rs is not None and ac_std != 0:
            a = (a.astype(np.float64) + rs.randn(a.shape[0]) * ac_std).astype(F32)
        ob, rew, done, _ = env.step(a)
        rews.append(rew)
        obs.append(ob)
        behv.extend(float(x) for x in env.pos)
        if done:
            break
    behv += behv[-3:] * (max_steps - len(behv) // 3)
    return rews, behv, np.array(obs), step


def episodes_fold(episode_rewards, max_steps: int):
    """obj.py:56-61: ``rews = zeros(max_steps); rews[:len(rew)] += rew`` per episode in order, ``rews /= E``."""
    rews = np.zeros(max_steps)
    for rew in episode_rewards:
        rews[:len(rew)] += np.array(rew)
    rews /= max(1, len(episode_rewards))
    return rews


def _env(T=40, h=None, obs=15, act=3, **kw):
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
    return ClosedLoopEnv(obs, act, T, band=4, fall_height=h, **kw)


def _policy(env, hidden=(16, 16), ac_std=0.0, seed=0, scale=1.0):
    from es_pytorch_b200.nn.nn import FeedForward
    torch.manual_seed(seed)
    m = FeedForward(list(hidden), torch.nn.Tanh(), env, ac_std)
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(scale)
    return m


# ---------------------------------------------------------------------------------------------- the done rule
def test_done_rule_is_float32_abs_z_after_the_update():
    env = _env(T=10, h=0.25, act=3, pos_scale=0.1)
    env.reset()
    a = np.array([0.0, 0.0, 1.0], F32)
    z = F32(0)
    for t in range(3):
        _, _, done, _ = env.step(a)
        z = F32(z + F32(F32(0.1) * F32(1.0)))
        assert env.pos[2] == z
        assert done == (not abs(z) <= F32(0.25)), t
    assert done                                          # 0.3 > 0.25 at the third step
    # h exactly |z|: stays; one float32 ulp below: falls; negative z counts by its magnitude
    for h, want in ((0.2, False), (float(np.nextafter(F32(0.2), F32(0))), True)):
        e = _env(T=10, h=h, pos_scale=0.1)
        e.reset()
        e.step(-a)
        _, _, done, _ = e.step(-a)
        assert e.pos[2] == F32(-0.2) and done == want, (h, done)


def test_nan_position_and_the_last_step_end_the_episode():
    env = _env(T=5, h=1e30)
    env.reset()
    _, _, done, _ = env.step(np.array([0.0, 0.0, np.nan], F32))
    assert done and np.isnan(env.pos[2])
    env = _env(T=3, h=1e30)
    env.reset()
    dones = [env.step(np.zeros(3, F32))[2] for _ in range(3)]
    assert dones == [False, False, True]


def test_no_fall_height_is_todays_env():
    a, b = _env(T=20), _env(T=20, h=1e30)
    assert a.fall_height is None and not a.terminates and b.terminates
    rs = np.random.RandomState(0)
    a.reset(); b.reset()
    for _ in range(20):
        act = rs.randn(3).astype(F32)
        ra, rb = a.step(act), b.step(act)
        assert np.array_equal(ra[0], rb[0]) and ra[1] == rb[1] and ra[2] == rb[2]


@pytest.mark.parametrize('bad', [0, 0.0, -1.0, float('nan'), float('inf'), 1e39])
def test_fall_height_must_be_finite_and_positive(bad):
    with pytest.raises(ValueError):
        _env(h=bad)


@pytest.mark.parametrize('bad', ['0.5', True, [0.5]])
def test_fall_height_must_be_a_number(bad):
    with pytest.raises(TypeError):
        _env(h=bad)


def test_gym_make_forwards_fall_height_and_the_open_loop_refuses_it():
    from es_pytorch_b200.gym import synthetic_env
    env = synthetic_env.make('HopperClosedLoop-v0', fall_height=0.5)
    assert env.fall_height == F32(0.5) and env.terminates
    with pytest.raises(TypeError):
        synthetic_env.make('Hopper-v0', fall_height=0.5)


# ---------------------------------------------------------------------------------------------- run_model's loop
def _restated(env, model, T):
    """run_model on the oracle's pieces: the oracle's closed-loop step, forward and float32 reward / position, the done
    rule of ClosedLoopEnv(fall_height)."""
    spec = orc.ClosedLoopEnvSpec(env.obs_dim, env.act_dim, env.T, band=env.band)
    sd = [p.detach().numpy().astype(F32) for p in model.parameters()]
    layers = [(sd[i], sd[i + 1]) for i in range(0, len(sd), 2)]
    mean, std = np.asarray(model._obmean, np.float64), np.asarray(model._obstd, np.float64)
    ob, pos = spec.obs_stream[0].copy(), np.zeros(3, F32)
    rews, behv, obs = [], [], []
    h = F32(env.fall_height)
    for t in range(T):
        a = orc.mlp_forward(layers, orc.normalise_obs(ob, mean, std, model.ob_clip)).astype(F32)
        acc = F32(0)
        for j in range(env.act_dim):
            acc = F32(acc + F32(a[j] * spec.rew_vec[t, j]))
        rews.append(float(acc))
        for j in range(3):
            pos[j] = F32(pos[j] + F32(F32(env.pos_scale) * a[j % env.act_dim]))
        behv += [float(x) for x in pos]
        ob = spec.step_obs(ob, a)
        obs.append(ob)
        if t == T - 1 or not abs(pos[2]) <= h:
            break
    behv += behv[-3:] * (T - len(behv) // 3)
    return rews, behv, np.array(obs), t


@pytest.mark.parametrize('h', [1e-4, 0.02, 0.06, 1e9])
def test_run_model_stops_where_the_restated_rule_does(h):
    from es_pytorch_b200.gym.gym_runner import run_model
    T = 60
    env = _env(T=T, h=h)
    model = _policy(env, scale=2.0, seed=1)
    got = run_model(model, env, T)
    want = _restated(env, model, T)
    assert got[3] == want[3] and len(got[0]) == want[3] + 1
    assert np.allclose(got[0], want[0], rtol=1e-5, atol=1e-6)
    assert np.allclose(got[1], want[1], rtol=1e-5, atol=1e-6) and len(got[1]) == 3 * T
    assert got[2].shape == (want[3] + 1, env.obs_dim) and np.allclose(got[2], want[2], atol=1e-5)
    if h == 1e9:
        assert got[3] == T - 1
    if h == 1e-4:
        assert got[3] == 0


def test_fold_of_episodes_where_the_last_is_shorter():
    """BatchedRollout's python route of obj.py:54-63 with action noise: each episode ends on its own, rews[:len] += rew, the
    mean over E; steps is the last episode's t_d.  The seed is one where the last episode is shorter than an earlier one."""
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    T, E = 50, 3
    env = _env(T=T, h=0.05)
    model = _policy(env, ac_std=0.3, seed=2)
    found = None
    for seed in range(200):
        rs = np.random.RandomState(seed)
        eps = [run_model(model, env, T, rs) for _ in range(E)]
        lens = [len(e[0]) for e in eps]
        if lens[-1] < max(lens[:-1]) and min(lens) < T:
            found = seed, eps
            break
    assert found is not None
    seed, eps = found
    want = episodes_fold([e[0] for e in eps], T)
    br = BatchedRollout(env, T, coins_per_eval=0, episodes=E)
    rs = np.random.RandomState(seed)
    rews, behv, steps = br._run_episodes(model, rs, E)
    assert np.array_equal(np.array(rews), want)
    assert steps == eps[-1][3] and behv == eps[-1][1]
    # the fold runs to the longest episode: steps beyond the last episode's end still carry the earlier ones' rewards
    assert np.any(np.array(rews)[len(eps[-1][0]):] != 0)


def test_restated_loop_matches_the_packages_run_model_with_noise():
    from es_pytorch_b200.gym.gym_runner import run_model
    T = 40
    env = _env(T=T, h=0.05)
    model = _policy(env, ac_std=0.2, seed=3)
    a, b = np.random.RandomState(4), np.random.RandomState(4)
    got = run_model(model, env, T, a)
    fwd = lambda ob: model(torch.from_numpy(np.asarray(ob)).float(), rs=None).detach().numpy()
    want = run_model_loop(env, fwd, T, b, 0.2)
    assert got[3] == want[3] and got[0] == want[0] and got[1] == want[1]
    sa, sb = a.get_state(), b.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def test_coin_words_are_the_words_random_consumes():
    """The per-evaluation route draws a save_obs coin as randint(0, 2^32, 2, uint32): the two words rs.random() consumes."""
    for seed in range(20):
        a, b = np.random.RandomState(seed), np.random.RandomState(seed)
        a.randn(seed % 3); b.randn(seed % 3)
        w = a.randint(0, 2 ** 32, size=2, dtype=np.uint32)
        assert orc.words_to_double(int(w[0]), int(w[1])) == b.random()
        sa, sb = a.get_state(), b.get_state()
        assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


# ---------------------------------------------------------------------------------------------- the float64 truth
def test_fall_height_nothing_reaches_is_no_fall_height():
    """closed_f64.simulate at h = 1e30 is its fall_height=None result bit for bit, for the truth and every modelled bug, with
    action noise over E = 3 episodes.  A NaN in ob_mean makes the position NaN from step 0: without a fall height every
    episode still runs T steps, with one every episode ends at step 0."""
    sizes, band, T, n, E = [15, 32, 32, 3], 4, 40, 3, 3
    act = sizes[-1]
    P = orc.n_params(orc.layer_dims(sizes[0], sizes[1:-1], act))
    rs = np.random.RandomState(6)
    table = rs.randn(P + 1000).astype(F32)
    theta = np.concatenate([rs.randn(fi * fo + fo) / np.sqrt(fi) for fi, fo in zip(sizes[:-1], sizes[1:])]).astype(F32)
    spec = orc.ClosedLoopEnvSpec(sizes[0], act, T, band=band)
    idx, mean, std = rs.randint(0, 1000, size=n), rs.randn(sizes[0]) * 0.05, 0.5 + rs.rand(sizes[0])
    args = lambda mean: (table, idx, theta, 0.02, sizes, mean, std, 1.0, spec.obs_stream[0].copy(),
                         np.ascontiguousarray(spec.env_a.T), np.ascontiguousarray(spec.env_b.T), spec.rew_vec, spec.pos_scale)
    kw = dict(act_noise=(rs.randn(n, 2, E * T * act) * 0.3).astype(F32), episodes=E)
    variants = [None] + cf.mutations(sizes, band, True, E)
    free = cf.simulate(*args(mean), variants=variants, **kw)
    high = cf.simulate(*args(mean), variants=variants, fall_height=1e30, **kw)
    assert free.keys() == high.keys()
    for k in free:
        if k != 'gap':                                   # |z - h|: inf without a height
            assert np.array_equal(free[k], high[k]), k
    assert (free['steps'] == T - 1).all() and (free['used'] == E * T * act).all()
    mean[1] = np.nan
    free, fall = cf.truth(*args(mean), **kw), cf.truth(*args(mean), fall_height=1e30, **kw)
    assert np.isnan(free['fit']).all() and np.isnan(free['z0']).all()
    assert (free['eps'] == T - 1).all() and (free['used'] == E * T * act).all()
    assert (fall['eps'] == 0).all() and (fall['used'] == E * act).all()


# ---------------------------------------------------------------------------------------------- C ABI
def test_terminal_entry_points_are_declared_and_bound():
    from es_pytorch_b200 import _lib, build
    build.build()
    hdr = open(os.path.join(ROOT, 'include', 'es_b200.h')).read()
    lib = _lib.load()
    for name in ('es_rollout_closedloop_terminal', 'es_fitness_objective_steps'):
        assert re.search(r'\b%s\s*\(' % name, hdr) and name in _lib.SIGNATURES and hasattr(lib, name)
        decl = re.search(r'\b%s\s*\(([^)]*)\)' % name, hdr).group(1)
        assert decl.count(',') + 1 == len(_lib.SIGNATURES[name][1]), name

