"""CPU oracle for multi-episode evaluations: obj.py's fit_fn with ``eps_per_policy`` episodes.

TEST INFRASTRUCTURE ONLY, built on ``oracle.es_oracle`` (which it leaves as it is).  The reference's main training script
averages ``cfg.general.eps_per_policy`` episodes per evaluation (obj.py:54-63)::

    save_obs = rs.random() < cfg.policy.save_obs_chance
    rews = np.zeros(cfg.env.max_steps)
    for _ in range(max(1, cfg.general.eps_per_policy)):
        rew, behv, obs, steps = gym_runner.run_model(model, env, cfg.env.max_steps, rs if use_ac_noise else None)
        rews[:len(rew)] += np.array(rew)
    rews /= max(1, cfg.general.eps_per_policy)
    return RewardResult(rews.tolist(), behv, obs if save_obs else zeros, steps)

``run_model_episodes`` restates that loop on top of ``es_oracle.run_model``.  ``es_test_params``, ``generation`` and
``es_step`` are es_oracle's with an ``episodes`` keyword: they run es_oracle's own functions with every evaluation's
``run_model`` call replaced by ``run_model_episodes`` (es_oracle looks ``run_model`` up in its module when it is called).
With ``episodes=1`` they ARE es_oracle's functions.  Behaviour, saved observations and ``steps`` are the last episode's.
"""
from __future__ import annotations

import contextlib

import numpy as np

from oracle import es_oracle as orc

_run_model = orc.run_model          # the single-episode rollout, captured before any rebinding


def run_model_episodes(env, layers, obmean, obstd, ob_clip: float, max_steps: int, batched: bool = False,
                       ac_std: float = 0.0, rs=None, episodes: int = 1):
    """obj.py:57-60: ``max(1, episodes)`` runs of run_model, each drawing its own action noise from ``rs`` (nn.py:47-48);
    the float32 rewards (python floats) summed per step into a float64 array in episode order, divided by the count."""
    n = max(1, int(episodes))
    rews = np.zeros(int(max_steps))
    for _ in range(n):
        rew, behv, obs, steps = _run_model(env, layers, obmean, obstd, ob_clip, max_steps, batched, ac_std, rs)
        rews[:len(rew)] += np.array(rew)
    rews /= n
    return rews.tolist(), behv, obs, steps


@contextlib.contextmanager
def _episodes(episodes: int):
    if max(1, int(episodes)) == 1:
        yield
        return

    def run_model(env, layers, obmean, obstd, ob_clip, max_steps, batched=False, ac_std=0.0, rs=None):
        return run_model_episodes(env, layers, obmean, obstd, ob_clip, max_steps, batched, ac_std, rs, episodes)

    orc.run_model = run_model
    try:
        yield
    finally:
        orc.run_model = _run_model


def es_test_params(*args, episodes: int = 1, **kw):
    """es_oracle.es_test_params with ``episodes`` episodes per evaluation."""
    with _episodes(episodes):
        return orc.es_test_params(*args, **kw)


def generation(*args, episodes: int = 1, **kw):
    """es_oracle.generation with ``episodes`` episodes per evaluation."""
    with _episodes(episodes):
        return orc.generation(*args, **kw)


def es_step(*args, episodes: int = 1, **kw):
    """es_oracle.es_step with ``episodes`` episodes per evaluation; the noiseless evaluation runs them too (obj.py's fit_fn
    loops whether or not it adds noise), which leaves its result unchanged."""
    with _episodes(episodes):
        return orc.es_step(*args, **kw)
