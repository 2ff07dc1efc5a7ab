"""Float64 truth of the closed-loop rollout on an env whose episodes end early (ClosedLoopEnv(fall_height=h),
es_rollout_closedloop_terminal), and a float32 restatement of run_model's loop on it.

TEST INFRASTRUCTURE ONLY.  ``truth`` takes the data the kernel gets and evaluates it as tests/closed_f64.py does (weights
``theta +- f64(sigma) eps``, ``clip((ob - mean) / std)``, the activation after every layer, the env ``tanh(A ob + B a)``), with
run_model's ``if done: break`` (src/gym/gym_runner.py:50-67) inside obj.py:54-63's episode loop:

* step t of an episode ends it when t = T - 1 or not |z_t| <= h, z_t the third position component after step t's update;
* the fitness is ``sum_t (sum_e r_{e,t}) / E`` over every step any episode executed; the reward mass likewise;
* episode e reads its action noise from where episode e - 1 stopped: the evaluation's noise is one flat run of E T act values
  of which the first ``sum_e (t_{d,e} + 1) act`` are used;
* behaviour, ObStat sums (t_d + 1 post-step rows) and t_d are the last episode's.

``gap``: per evaluation, the smallest | |z_t| - h | over the executed steps of every episode: an implementation whose position
is off by less than that decides every step's fall as the truth does.  ``margin``: for a binned head, the smallest gap between
a dimension's two largest outputs over the executed steps (an arg-max that close is a knife edge).
"""
from __future__ import annotations

import os
import sys
from typing import Optional

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closed_f64 as cf  # noqa: E402

F32 = np.float32


def truth(table, idx, theta, sigma, sizes, ob_mean, ob_std, clip, obs0, env_a, env_b, rew_vec, pos_scale, fall_height,
          act_noise=None, episodes: int = 1, activation=np.tanh, binned=None):
    """Returns a dict indexed [2][n] (sign, pair): 'fit', 'mass', 'steps' (the last episode's t_d), 'used' (noise values
    consumed), 'eps' ([..][E] every episode's t_d), 'gap', 'margin', 'zmax' (the largest |z| reached), 'z0' (|z| after the last
    episode's first step), and [2][n][k] 'behv', 'mag' (3), 'osum', 'osq',
    'oabs' (obs).  ``binned``: (bins, low, high) of an FFBinned head (the last layer's outputs are adim * bins).
    ``act_noise``: [n][2][E T act] (or any shape of that size) scaled float32 gaussians."""
    idx = np.asarray(idx)
    n = len(idx)
    N, E = 2 * n, int(episodes)
    T = rew_vec.shape[0]
    layers = cf._weights(table, idx, theta, sigma, sizes, range(n))
    L = len(layers)
    c = np.asarray(rew_vec, np.float64)
    act = c.shape[1]
    B = np.asarray(env_b, np.float64)
    A = cf._env_matrix(env_a, sizes[0]).T.copy()
    mean, std = np.asarray(ob_mean, np.float64), np.asarray(ob_std, np.float64)
    ps, h = float(F32(pos_scale)), float(F32(fall_height))
    nz = None if act_noise is None else np.asarray(act_noise, np.float32).reshape(N, -1).astype(np.float64)
    rows = np.arange(N)
    cols = [0, 1 % act, 2 % act]
    rew_sum, mass_sum = np.zeros((N, T)), np.zeros((N, T))
    used = np.zeros(N, np.int64)
    eps = np.zeros((N, E), np.int64)
    gap, margin = np.full(N, np.inf), np.full(N, np.inf)
    zmax, z0 = np.zeros(N), np.zeros(N)
    for e in range(E):
        ob = np.broadcast_to(np.asarray(obs0, np.float64), (N, sizes[0])).copy()
        pos, mag = np.zeros((N, 3)), np.zeros((N, 3))
        osum, osq, oabs = (np.zeros((N, sizes[0])) for _ in range(3))
        alive = np.ones(N, bool)
        t_d = np.full(N, T - 1, np.int64)
        for t in range(T):
            if not alive.any():
                break
            x = cf.normalise(ob, mean, std, clip)
            for l, (WT, b, _) in enumerate(layers):
                z = np.einsum('ni,nio->no', x, WT) + b
                x = np.tanh(z) if (binned is not None or activation is None) else activation(z)
            if binned is not None:
                bins, low, high = binned
                out = x.reshape(N, -1, bins)
                top = np.sort(out, axis=2)
                margin = np.where(alive, np.minimum(margin, (top[:, :, -1] - top[:, :, -2]).min(axis=1)), margin)
                lo = np.asarray(low, np.float64)
                a = lo + (np.asarray(high, np.float64) - lo) * out.argmax(axis=2) / (bins - 1.0)
            else:
                a = x
            if nz is not None:
                a = a + nz[rows[:, None], used[:, None] + t * act + np.arange(act)[None, :]]
            prod = a * c[t]
            rew_sum[:, t] += np.where(alive, prod.sum(axis=1), 0.0)
            mass_sum[:, t] += np.where(alive, np.abs(prod).sum(axis=1), 0.0)
            term = ps * a[:, cols]
            npos = pos + term
            nob = np.tanh(ob @ A + a @ B)
            lv = alive[:, None]
            mag = np.where(lv, mag + np.abs(npos) + np.abs(term), mag)
            pos = np.where(lv, npos, pos)
            ob = np.where(lv, nob, ob)
            osum += ob * lv
            osq += ob * ob * lv
            oabs += np.abs(ob) * lv
            gap = np.where(alive, np.minimum(gap, np.abs(np.abs(pos[:, 2]) - h)), gap)
            zmax = np.where(alive, np.maximum(zmax, np.abs(pos[:, 2])), zmax)
            if t == 0:
                z0 = np.abs(pos[:, 2])
            ended = alive & (~(np.abs(pos[:, 2]) <= h) | (t == T - 1))
            t_d[ended] = t
            alive &= ~ended
        eps[:, e] = t_d
        used += (t_d + 1) * act
    res = dict(fit=rew_sum.sum(axis=1) / E, mass=mass_sum.sum(axis=1) / E, steps=t_d, used=used, eps=eps, gap=gap,
               margin=margin, zmax=zmax, z0=z0, behv=pos, mag=mag, osum=osum, osq=osq, oabs=oabs)

    def shape(v):                                              # [N][...] (pair-major, + then -) -> [2][n][...]
        return np.swapaxes(v.reshape((n, 2) + v.shape[1:]), 0, 1)
    return {k: shape(v) for k, v in res.items()}


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
