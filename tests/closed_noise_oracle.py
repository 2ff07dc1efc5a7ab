"""CPU oracle for the closed-loop synthetic env with action noise and multi-episode evaluations.

TEST INFRASTRUCTURE ONLY, built on ``oracle.es_oracle`` (which it leaves as it is).  ``es_oracle.run_model`` defines the
closed-loop env without action noise; this module restates its literal per-step loop (gym_runner.py:33-67 with
FeedForward.forward, nn.py:42-50) with the noise the reference adds at every step::

    a = forward(clip((ob - mean) / std))
    a = float32(float64(a) + rs.randn(act) * ac_std)        # a float32 tensor plus a float64 ndarray, cast by the env
    reward = <a, c_t> (float32, index order); pos += pos_scale * a[0..2]; ob = step_obs(ob, a)

and obj.py:54-63's ``eps_per_policy`` loop on top of it: E episodes from a fresh env, the rewards summed per step in float64
in episode order and divided by E; behaviour, observations and ``steps`` are the last episode's.  ``es_test_params``,
``generation`` and ``es_step`` are es_oracle's with every evaluation's ``run_model`` call replaced while they run (es_oracle
looks ``run_model`` up in its module when it is called).
"""
from __future__ import annotations

import contextlib

import numpy as np

from oracle import es_oracle as orc

F32 = np.float32
_run_model = orc.run_model          # the single-episode rollout, captured before any rebinding


def run_model_closed(env, layers, obmean, obstd, ob_clip: float, max_steps: int, ac_std: float = 0.0, rs=None):
    """One episode of ``orc.run_model_closed``'s loop with the action noise drawn from ``rs`` at every step (none when
    ``ac_std == 0`` or ``rs`` is None, as nn.py:47)."""
    n = min(int(max_steps), env.T)
    rews, behv, obs = [], [], []
    pos = np.zeros(3, dtype=F32)
    ps = F32(env.pos_scale)
    ob = env.obs_stream[0].copy()
    for t in range(n):
        a = orc.mlp_forward(layers, orc.normalise_obs(ob, obmean, obstd, ob_clip)).astype(F32)
        if ac_std != 0 and rs is not None:
            a = (a.astype(np.float64) + rs.randn(env.act_dim) * ac_std).astype(F32)
        acc = F32(0.0)
        for j in range(env.act_dim):           # float32 dot, index order
            acc = F32(acc + F32(a[j] * env.rew_vec[t, j]))
        rews.append(float(acc))
        for j in range(3):
            pos[j] = F32(pos[j] + F32(ps * a[j % env.act_dim]))
        behv.extend([float(pos[0]), float(pos[1]), float(pos[2])])
        ob = env.step_obs(ob, a)
        obs.append(ob)
    step = n - 1
    behv += behv[-3:] * (max_steps - int(len(behv) / 3))
    return rews, behv, np.stack(obs), step


def run_model_episodes(env, layers, obmean, obstd, ob_clip: float, max_steps: int, ac_std: float = 0.0, rs=None,
                       episodes: int = 1):
    """obj.py:57-60 on the closed loop: ``max(1, episodes)`` episodes, each from obs_0 and drawing its own noise."""
    n = max(1, int(episodes))
    rews = np.zeros(int(max_steps))
    for _ in range(n):
        rew, behv, obs, steps = run_model_closed(env, layers, obmean, obstd, ob_clip, max_steps, ac_std, rs)
        rews[:len(rew)] += np.array(rew)
    rews /= n
    return rews.tolist(), behv, obs, steps


@contextlib.contextmanager
def _closed_noise(episodes: int):
    def run_model(env, layers, obmean, obstd, ob_clip, max_steps, batched=False, ac_std=0.0, rs=None):
        if getattr(env, 'closed_loop', False):
            return run_model_episodes(env, layers, obmean, obstd, ob_clip, max_steps, ac_std, rs, episodes)
        return _run_model(env, layers, obmean, obstd, ob_clip, max_steps, batched, ac_std, rs)

    orc.run_model = run_model
    try:
        yield
    finally:
        orc.run_model = _run_model


def es_test_params(*args, episodes: int = 1, **kw):
    """es_oracle.es_test_params on the closed loop with action noise (``ac_std=``) and ``episodes`` episodes per evaluation."""
    with _closed_noise(episodes):
        return orc.es_test_params(*args, **kw)


def generation(*args, episodes: int = 1, **kw):
    """es_oracle.generation, as ``es_test_params``."""
    with _closed_noise(episodes):
        return orc.generation(*args, **kw)


def es_step(*args, episodes: int = 1, **kw):
    """es_oracle.es_step, as ``es_test_params``; its noiseless evaluation draws no noise and its episodes are identical."""
    with _closed_noise(episodes):
        return orc.es_step(*args, **kw)
