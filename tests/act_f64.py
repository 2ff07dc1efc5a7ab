"""Float64 truth of the rollouts for policies with any activation: what es_rollout_*_activation approximates.

TEST INFRASTRUCTURE ONLY.  The same definitions as f64_rollout (open loop) and closed_f64 (closed loop, unmutated), with the
policy's activation a float64 function in place of tanh after every layer; the closed-loop env's own tanh stays.  With
``np.tanh`` both reproduce those modules to 1e-13 relative (tests/test_activations_host.py checks it), so the bounds built on them
carry over.  Layouts, units and the returned arrays are theirs.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import closed_f64
import f64_rollout as f64


# ---- the float64 forms of the activations (parameters as float32 values, as the kernels and torch take them)
def leaky_relu(slope: float):
    s = float(np.float32(slope))
    return lambda z: np.where(z > 0, z, z * s)


def elu(alpha: float):
    a = float(np.float32(alpha))
    return lambda z: np.where(z > 0, z, a * np.expm1(z))


def relu(z):
    return np.maximum(z, 0.0)


def sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


def form(activation, xp=np):
    """The float64 form of an ``nn.Activation`` (None: tanh) -- the functions above -- for numpy arrays, or with
    ``xp=torch`` the same forms for torch.float64 tensors."""
    from es_pytorch_b200 import _lib
    kind = _lib.ES_ACT_TANH if activation is None else int(activation.kind)
    p = 0.0 if activation is None else float(np.float32(activation.param))
    if xp is np:
        return {_lib.ES_ACT_TANH: np.tanh, _lib.ES_ACT_RELU: relu, _lib.ES_ACT_LEAKY_RELU: leaky_relu(p),
                _lib.ES_ACT_ELU: elu(p), _lib.ES_ACT_SIGMOID: sigmoid}[kind]
    return {_lib.ES_ACT_TANH: xp.tanh, _lib.ES_ACT_RELU: lambda z: xp.clamp_min(z, 0.0),
            _lib.ES_ACT_LEAKY_RELU: lambda z: xp.where(z > 0, z, z * p),
            _lib.ES_ACT_ELU: lambda z: xp.where(z > 0, z, p * xp.expm1(z)),
            _lib.ES_ACT_SIGMOID: lambda z: 1.0 / (1.0 + xp.exp(-z))}[kind]


def per_layer(activation, n_layers: int) -> list:
    """``activation`` for each of ``n_layers`` layers: a sequence of one function per layer as it is, one function repeated."""
    acts = list(activation) if isinstance(activation, (list, tuple)) else [activation] * n_layers
    assert len(acts) == n_layers, (len(acts), n_layers)
    return acts


def episode(w, layer_sizes, obsn, rew_vec, pos_scale, activation, noise: Optional[np.ndarray] = None):
    """f64_rollout.episode with ``activation`` after every layer (or a list of one function per layer)."""
    a = obsn.astype(np.float64)
    lay = f64.layer_slices(layer_sizes)
    for (wo, bo, fi, fo), act_fn in zip(lay, per_layer(activation, len(lay))):
        a = act_fn(a @ w[wo:wo + fi * fo].reshape(fo, fi).T + w[bo:bo + fo])
    c = rew_vec.astype(np.float64)
    act = a.shape[1]
    if noise is None:
        noise = np.zeros((1,) + a.shape, dtype=np.float32)
    rew, rabs = np.zeros(a.shape[0]), np.zeros(a.shape[0])
    for nz in noise:
        an = a + nz.astype(np.float64)
        rew += (an * c).sum(axis=1)
        rabs += np.abs(an * c).sum(axis=1)
    rew /= len(noise)
    rabs /= len(noise)
    terms = float(pos_scale) * an[:, [j % act for j in range(3)]]
    behv = terms.sum(axis=0)
    mag = np.abs(np.cumsum(terms, axis=0)).sum(axis=0) + np.abs(terms).sum(axis=0)
    return rew, rabs, behv, mag


def rollout_f64(table, idx, theta, sigma, layer_sizes, obsn, rew_vec, pos_scale, activation, act_noise=None, episodes: int = 1,
                pairs: Optional[Sequence[int]] = None):
    """f64_rollout.rollout_f64 with ``activation``: (fitness [2, n], behaviour [2, n, 3], reward mass [2, n], position
    magnitude [2, n, 3])."""
    idx = np.asarray(idx)
    pairs = range(len(idx)) if pairs is None else pairs
    T, act = rew_vec.shape
    fit, mass = np.zeros((2, len(pairs))), np.zeros((2, len(pairs)))
    behv, mag = np.zeros((2, len(pairs), 3)), np.zeros((2, len(pairs), 3))
    for n, k in enumerate(pairs):
        for s, sign in enumerate((1.0, -1.0)):
            nz = None if act_noise is None else np.asarray(act_noise[k, s]).reshape(episodes, T, act)
            r, ra, b, m = episode(f64.perturbed(table, idx[k], theta, sigma, sign), layer_sizes, obsn, rew_vec, pos_scale,
                                  activation, nz)
            fit[s, n], behv[s, n], mass[s, n], mag[s, n] = r.sum(), b, ra.sum(), m
    return fit, behv, mass, mag


def closed_truth(table, idx, theta, sigma, sizes, ob_mean, ob_std, clip, obs0, env_a, env_b, rew_vec, pos_scale,
                 act_noise=None, episodes: int = 1, activation=np.tanh):
    """closed_f64.truth (no mutation) with the policy's ``activation`` (or a list of one per layer): a dict of float64 arrays indexed [2][n] ([2][n][...]
    for vectors): 'fit', 'mass', 'behv', 'mag', 'osum', 'osq', 'oabs' (the last episode's, as the kernels keep them)."""
    idx = np.asarray(idx)
    n = len(idx)
    T, act = rew_vec.shape
    obs, E, N = sizes[0], int(episodes), 2 * n
    layers = closed_f64._weights(table, idx, theta, sigma, sizes, range(n))
    c = np.asarray(rew_vec, np.float64)
    B = np.asarray(env_b, np.float64)                      # [act][obs]: pre += a @ B
    A = closed_f64._env_matrix(env_a, obs).T.copy()        # pre += ob @ A
    mean, std = np.asarray(ob_mean, np.float64), np.asarray(ob_std, np.float64)
    ps = float(np.float32(pos_scale))
    nz_all = None
    if act_noise is not None:
        nz_all = np.asarray(act_noise, np.float32).reshape(N, E, T, act).astype(np.float64)
    cols = [0, 1 % act, 2 % act]
    fit, mass = np.zeros(N), np.zeros(N)
    for e in range(E):
        ob = np.broadcast_to(np.asarray(obs0, np.float64), (N, obs)).copy()
        pos, mag = np.zeros((N, 3)), np.zeros((N, 3))
        osum, osq, oabs = (np.zeros((N, obs)) for _ in range(3))
        for t in range(T):
            h = closed_f64.normalise(ob, mean, std, float(clip))
            for (WT, b, _), act_fn in zip(layers, per_layer(activation, len(layers))):
                h = act_fn(np.matmul(h[:, None, :], WT)[:, 0, :] + b)
            a = h if nz_all is None else h + nz_all[:, e, t]
            prod = a * c[t]
            fit += prod.sum(axis=1) / E
            mass += np.abs(prod).sum(axis=1) / E
            term = ps * a[:, cols]
            pos = pos + term
            mag += np.abs(pos) + np.abs(term)
            ob = np.tanh(ob @ A + a @ B)                   # the env's own tanh
            osum += ob
            osq += ob * ob
            oabs += np.abs(ob)
    res = dict(fit=fit, mass=mass, behv=pos, mag=mag, osum=osum, osq=osq, oabs=oabs)
    return {k: v.reshape((n, 2) + v.shape[1:]).swapaxes(0, 1) for k, v in res.items()}
