"""CPU oracle for binned-action policies: the reference's ``FFBinned`` (src/nn/nn.py:99-117) on the synthetic envs.

TEST INFRASTRUCTURE ONLY, built on ``oracle.es_oracle`` (which it leaves as it is).  FFBinned's forward is FeedForward's
Linear + Tanh stack with ``adim * bins`` outputs, followed by::

    ac_range = (self.ahigh - self.alow)[None, :]
    binned_ac = a.reshape((-1, self.adim, self.bins)).argmax(2)
    return (1. / (self.bins - 1.) * binned_ac * ac_range + self.alow[None, :]).squeeze()

With float32 ``low`` / ``high`` (the env's Box) torch evaluates this as ``((c * idx) * range) + low`` with
``c = float32(1 / (bins - 1))`` and every operation rounded to float32 (``binned_action``; tests/test_binned_host.py checks it
against ``FFBinned.forward`` for every idx with bins 2 to 32).  The forward draws no random numbers, so ``run_model`` is
es_oracle's ``run_model`` / ``run_model_closed`` (``ac_std == 0``) with ``forward``, the binned forward, in place of the tanh
stack's: the same normalisation, env steps, float32 reward dot, position integrator and outputs.  Nothing in es_oracle is
rebound.
"""
from __future__ import annotations

import numpy as np

from oracle import es_oracle as orc

F32 = np.float32


def binned_action(out: np.ndarray, bins: int, low: np.ndarray, high: np.ndarray) -> np.ndarray:
    """[..., adim * bins] network outputs -> [..., adim] float32 actions: the first maximal bin of each dimension (numpy's
    argmax, like torch's, returns the first), then ``((c * idx) * range) + low`` in float32."""
    out = np.asarray(out, dtype=F32)
    low = np.asarray(low, dtype=F32)
    rng = (np.asarray(high, dtype=F32) - low).astype(F32)
    idx = out.reshape(out.shape[:-1] + (low.shape[0], int(bins))).argmax(-1)
    c = F32(1.0 / (bins - 1.0))
    return (((c * idx.astype(F32)).astype(F32) * rng).astype(F32) + low).astype(F32)


def forward(layers, x: np.ndarray, bins: int, low, high) -> np.ndarray:
    """FFBinned.forward on normalised float32 inputs ``x`` ([obs] or [B, obs]): the tanh stack, then the binned head."""
    return binned_action(orc.mlp_forward(layers, x), bins, low, high)


def _step_outputs(env, t: int, a: np.ndarray, pos: np.ndarray, rews: list, behv: list):
    """es_oracle's per-step reward (float32 dot, index order) and position update for the action ``a``."""
    acc = F32(0.0)
    for j in range(env.act_dim):
        acc = F32(acc + F32(a[j] * env.rew_vec[t, j]))
    rews.append(float(acc))
    ps = F32(env.pos_scale)
    for j in range(3):
        pos[j] = F32(pos[j] + F32(ps * a[j % env.act_dim]))
    behv.extend([float(pos[0]), float(pos[1]), float(pos[2])])


def run_model(env, layers, obmean, obstd, ob_clip: float, max_steps: int, bins: int, low, high, batched: bool = False):
    """es_oracle.run_model (open loop) / run_model_closed (an env with ``closed_loop``) for a binned policy: (rews, behv
    padded to max_steps triples, post-step observations, last loop index).  ``batched``: the open loop's forward for all steps
    at once (the decisions are the per-step ones wherever the float64 truth's top two bins are apart)."""
    n = min(int(max_steps), env.T)
    rews, behv, pos = [], [], np.zeros(3, dtype=F32)
    if getattr(env, 'closed_loop', False):
        ob, obs = env.obs_stream[0].copy(), []
        for t in range(n):
            a = forward(layers, orc.normalise_obs(ob, obmean, obstd, ob_clip), bins, low, high)
            _step_outputs(env, t, a, pos, rews, behv)
            ob = env.step_obs(ob, a)
            obs.append(ob)
        obs = np.stack(obs)
    else:
        xs = orc.normalise_obs(env.obs_stream[:n], obmean, obstd, ob_clip)
        acts = forward(layers, xs, bins, low, high) if batched else np.stack([forward(layers, xs[t], bins, low, high)
                                                                              for t in range(n)])
        for t in range(n):
            _step_outputs(env, t, acts[t], pos, rews, behv)
        obs = env.obs_stream[1:n + 1].copy()
    behv += behv[-3:] * (max_steps - int(len(behv) / 3))
    return rews, behv, obs, n - 1


def raw_outputs_f64(layers, x: np.ndarray) -> np.ndarray:
    """The float64 truth of the tanh stack's outputs ([..., adim * bins]) for float32 inputs ``x``."""
    h = np.asarray(x, dtype=np.float64)
    for w, b in layers:
        h = np.tanh(h @ np.asarray(w, np.float64).T + np.asarray(b, np.float64))
    return h


def top_two_gap(out: np.ndarray, bins: int) -> float:
    """The smallest gap between the largest and the second largest output of any action dimension's bins in ``out``
    ([..., adim * bins]): the margin by which every arg-max decision is taken."""
    o = np.sort(np.asarray(out).reshape(-1, int(bins)), axis=1)
    return float((o[:, -1] - o[:, -2]).min())


def closed_inputs(env, layers, obmean, obstd, ob_clip: float, max_steps: int, bins: int, low, high) -> np.ndarray:
    """The normalised observations [T, obs] the oracle's closed-loop episode of the binned policy feeds its network."""
    n = min(int(max_steps), env.T)
    ob = env.obs_stream[0].copy()
    xs = []
    for _ in range(n):
        x = orc.normalise_obs(ob, obmean, obstd, ob_clip)
        xs.append(x)
        ob = env.step_obs(ob, forward(layers, x, bins, low, high))
    return np.stack(xs)
