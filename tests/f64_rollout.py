"""Float64 reference of the open-loop rollout: what every device rollout mode approximates.

TEST INFRASTRUCTURE ONLY.  It takes the float32 data the kernels get and evaluates them in float64 without intermediate
rounding, so a kernel can be judged on its own rather than against another float32 implementation:

* the weights are ``theta +- f64(sigma) * eps`` exactly (``sigma`` is passed to the kernels as a float32), any number of
  layers, state-dict flat layout (``weight[out, in]`` row-major, then ``bias[out]``, layer after layer);
* every layer is ``activation(x W^T + b)`` over the whole episode as one float64 matrix product, tanh unless the policy
  has another activation (the float64 forms below, parameters as the float32 values the kernels and torch take);
* episode ``e`` acts ``a_t + nz_e,t`` (``act_noise`` [n_pairs, 2, E, T, act], the scaled float32 gaussians) and earns
  ``<a, c_t>``; the step's reward is the mean over the episodes and the fitness is its sum over t;
* the reward mass ``sum_t mean_e sum_j |a_tj c_tj|`` is the scale of the fitness error of any implementation whose actions
  carry a relative error: a float32 dot product is within ``act * 2^-24`` of it per step and an action error ``d`` moves it
  by at most ``d`` times it.  It bounds ``sum_t |r_t|`` from above and equals it unless the products of one step cancel
  (a single step can earn ~0 from large products);
* the behaviour is the last episode's ``pos_scale * sum_t a_t[i % act]`` for i = 0, 1, 2.

The observations ``obsn`` are taken as given: normalisation happens before the rollout and has its own bit-exact tests.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np


def layer_slices(layer_sizes: Sequence[int]):
    """[(w_off, b_off, n_in, n_out)] of every layer in the flat parameter vector."""
    out, off = [], 0
    for fi, fo in zip(layer_sizes[:-1], layer_sizes[1:]):
        out.append((off, off + fi * fo, fi, fo))
        off += fi * fo + fo
    return out


def n_params(layer_sizes: Sequence[int]) -> int:
    return sum(fi * fo + fo for fi, fo in zip(layer_sizes[:-1], layer_sizes[1:]))


def perturbed(table: np.ndarray, i: int, theta: np.ndarray, sigma: float, sign: float) -> np.ndarray:
    """theta + sign * f64(f32(sigma)) * table[i : i + P], exact in float64."""
    P = len(theta)
    s = float(np.float32(sigma))
    return theta.astype(np.float64) + sign * s * table[int(i):int(i) + P].astype(np.float64)


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


def episode(w: np.ndarray, layer_sizes: Sequence[int], obsn: np.ndarray, rew_vec: np.ndarray, pos_scale: float,
            noise: Optional[np.ndarray] = None, activation=np.tanh):
    """One evaluation of the flat float64 weights ``w``.  ``noise``: [E, T, act] or None (one noiseless episode).
    ``activation``: the policy's float64 activation after every layer, or a list of one per layer.
    Returns (per-step reward [T] (mean over the episodes), its mass sum_j |a_tj c_tj| [T] (mean over the episodes),
    behaviour [3], position magnitude [3]), all float64.  The
    magnitude is sum_t |partial sum_t| + sum_t |term_t| of each position component: a float32 sum of those terms in step
    order is within 2^-24 times it of the exact sum (to first order), which is what the position checks build on."""
    a = obsn.astype(np.float64)
    lay = layer_slices(layer_sizes)
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


def rollout_f64(table, idx, theta, sigma, layer_sizes, obsn, rew_vec, pos_scale, act_noise=None, episodes: int = 1,
                pairs: Optional[Sequence[int]] = None, activation=np.tanh):
    """The truth of ``Engine.rollout`` for the pairs ``pairs`` (default: all), with ``activation`` as ``episode`` takes it.
    Returns float64 arrays (fitness [2, n], behaviour [2, n, 3], reward mass [2, n], position magnitude [2, n, 3]) with
    row 0 the +eps and row 1 the -eps evaluation."""
    idx = np.asarray(idx)
    pairs = range(len(idx)) if pairs is None else pairs
    T, act = rew_vec.shape
    fit, mass = np.zeros((2, len(pairs))), np.zeros((2, len(pairs)))
    behv, mag = np.zeros((2, len(pairs), 3)), np.zeros((2, len(pairs), 3))
    for n, k in enumerate(pairs):
        for s, sign in enumerate((1.0, -1.0)):
            nz = None if act_noise is None else np.asarray(act_noise[k, s]).reshape(episodes, T, act)
            r, ra, b, m = episode(perturbed(table, idx[k], theta, sigma, sign), layer_sizes, obsn, rew_vec, pos_scale, nz,
                                  activation)
            fit[s, n], behv[s, n], mass[s, n], mag[s, n] = r.sum(), b, ra.sum(), m
    return fit, behv, mass, mag
