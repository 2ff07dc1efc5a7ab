"""Float64 reference of the closed-loop rollout (es_rollout_closedloop_mlp / _episodes / _terminal): what every closed-loop
kernel approximates.

TEST INFRASTRUCTURE ONLY.  It takes the data the kernels get and evaluates them in float64 without intermediate rounding:

* the weights are ``theta +- f64(sigma) * eps`` exactly (``sigma`` as the float32 the kernels receive), state-dict layout;
* every step normalises the raw observation, ``clip((ob - mean) / std, -clip, clip)``, runs ``activation(W x + b)`` after
  every layer (tanh, or f64_rollout's float64 forms of the other activations; a binned head, ``binned = (bins, low, high)``,
  runs tanh and takes each action dimension's arg-max in bin order, ``low + (high - low) bin / (bins - 1)``), adds the
  episode's action noise ``nz`` (``act_noise`` [n_pairs][2][E T act], the scaled float32 gaussians), earns ``<a + nz, c_t>``,
  integrates the position ``pos_scale * (a + nz)[i % act]`` and steps the env,
  ``ob_i <- tanh(sum_d A[i, d] ob[(i + d - half) mod n] + sum_j B[i, j] (a + nz)_j)``;
* with ``fall_height`` h (ClosedLoopEnv(fall_height=h)), step t ends an episode when t = T - 1 or not |z_t| <= f32(h), z_t
  the third position component after step t's update, so a NaN position ends it too (run_model's ``if done: break``
  inside obj.py's episode loop); without one every episode runs T steps whatever the position;
* every episode restarts from ``obs0`` with the position at 0 and reads its noise from the evaluation's flat run where the
  previous episode stopped (offset ``used + t act``); the fitness is ``sum_t (sum_e r_{e,t}) / E`` over the executed steps,
  the reward mass ``sum_t (sum_e sum_j |a_tj c_tj|) / E`` (the scale of the fitness error of an implementation whose actions
  carry a relative error, as in f64_rollout.py);
* behaviour, position magnitude (f64_rollout.episode's), the float64 column sums of the post-step observations and of their
  squares (the ObStat increments), the final observation ``olast`` and the last executed step t_d are the last episode's.

The evaluations of a call are stacked, so that a step is one batched matrix product per layer; so are *variants* of every
evaluation: ``simulate(variants=)`` runs, beside the truth, copies of it computed wrongly on purpose (the bugs a kernel could have, see
``MUTATIONS``), and ``growth`` runs copies whose start observation is moved by 1e-9.  One step loop with an alive mask runs
every episode, so an env where nothing falls gives the fixed-length result by construction.  Nothing here imports the
kernels.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import f64_rollout as f64

U = 2.0 ** -24
TANH_APPROX = 2.0 ** -11            # the relative error of tanh.approx.f32

# The bounds a closed-loop kernel is held to against this truth (tests/test_gpu_closed_f64.py explains and measures them):
EVAL_REL = 1e-5                     # per evaluation |f - truth| <= EVAL_REL * mass
RMS_BOUND = 3e-4                    # over the evaluations rms(f - truth) <= RMS_BOUND * spread
ACT_ERR = 1e-5                      # the error of one action, in the position bound 2 U mag + ACT_ERR pos_scale T
OBS_ERR = 1e-6                      # the error of one observation, in the ObStat bounds


# ---------------------------------------------------------------------------------------------- the cluster kernel's plan, restated
def _pad32(n):
    return (n + 31) & ~31


def _pad4(n):
    return (n + 3) & ~3


def one_cta_covers(sizes: Sequence[int]) -> bool:
    """api.cu's es_closed_one_cta_covers: rollout_closed.cu's one CTA per pair."""
    return len(sizes) == 4 and max(sizes[1:]) <= 64 and sizes[0] <= 384


def cluster_size(sizes: Sequence[int], band: int) -> Optional[int]:
    """rollout_closedw.cu's cw_plan: the smallest C in {1, 2, 4, 8} whose cw_layout fits 227 KiB - 1 KiB per CTA (None: no C
    fits).  The checks of the shape itself (layer count, widths, obs, act, band) are not restated."""
    obs, act, L = sizes[0], sizes[-1], len(sizes) - 1
    for C in (1, 2, 4, 8):
        at = 4 * obs + 8 + _pad32(obs) + sum(_pad32(d) for d in sizes[1:])
        for l in range(L):
            rows = -(-sizes[l + 1] // C)
            at += _pad4(rows) * _pad32(sizes[l]) + _pad4(rows)
        at += _pad4(act) + 2 * obs + 2 * _pad4(obs + 16) + _pad4(band * obs) + _pad4(act * obs)
        if 4 * at <= 227 * 1024 - 1024:
            return C
    return None


def plan(sizes: Sequence[int], band: int) -> int:
    """CTAs per cluster as Engine.closed_mlp_plan reports it: 0 for the one-CTA kernel."""
    return 0 if one_cta_covers(sizes) else cluster_size(sizes, band)


def owned_row_edges(sizes: Sequence[int], band: int):
    """[(layer, row)]: the first and the last output row of every layer that a CTA owns (rows [q R_l, min((q + 1) R_l, d)) for
    R_l = ceil(d / C)); rows 0 and d - 1 on the one-CTA kernel."""
    C = plan(sizes, band)
    out = set()
    for l, d in enumerate(sizes[1:]):
        if C == 0:
            out |= {(l, 0), (l, d - 1)}
            continue
        R = -(-d // C)
        for q in range(C):
            if q * R < d:
                out |= {(l, q * R), (l, min((q + 1) * R, d) - 1)}
    return sorted(out)


# ---------------------------------------------------------------------------------------------- mutations
def mutations(sizes: Sequence[int], band: int, noisy: bool, episodes: int):
    """Every bug ``simulate(variants=)`` models that applies to this shape and run: tuples (name, *args)."""
    L = len(sizes) - 1
    out = [('row', l, r) for l, r in owned_row_edges(sizes, band)]
    out += [('col', l, k) for l in range(L) for k in sorted({sizes[l] - 1, 32}) if k < sizes[l]]
    out += [('stale', l) for l in range(1, L)]
    out += [('band_shift',), ('band_nowrap',), ('b_last_col',)]
    out += [('no_clip',), ('no_mean',)]
    out += [('bias', l) for l in range(L)]
    out += [('drop_last_step',), ('skip_first_env_step',), ('tanh_approx',)]
    if noisy:
        out += [('env_clean',), ('rew_clean',), ('swap_sign_noise',)]
        if episodes > 1:
            out += [('ep0_noise',)]
    if episodes > 1:
        out += [('no_reset_obs',), ('no_reset_pos',), ('first_episode_outputs',)]
    return out


MUTATIONS = """\
row l r            layer l's output row r is never written (reads as 0: the buffers start zeroed)
col l k            layer l skips input column k
stale l            layer l >= 1 reads the previous step's activations of layer l - 1 (0 at the first step)
band_shift         the env's band is read one observation further: ob[(i + d - half + 1) mod n]
band_nowrap        the band does not wrap around: neighbours outside [0, n) read as 0
b_last_col         the env step misses B's last column
no_clip / no_mean  the normalisation does not clip / does not subtract the mean
bias l             layer l's bias is theta's, not perturbed
drop_last_step     the last step (reward, position, env step) is not taken
skip_first_env_step  the env does not step at t = 0 (the observation stays obs_0)
tanh_approx        every tanh is off by a relative 2^-11 (tanh.approx.f32's grade)
env_clean / rew_clean  the env step / the reward (and position) use the noise-free action
swap_sign_noise    the + evaluation takes the - evaluation's noise run and vice versa (each at its own offset)
ep0_noise          every episode reads its noise from offset 0, where episode 0 does
no_reset_obs / no_reset_pos  an episode after the first continues from the previous one's last observation / position
first_episode_outputs  behaviour and ObStat come from the first episode instead of the last
"""


# ---------------------------------------------------------------------------------------------- the simulator
def _env_matrix(env_a: np.ndarray, n: int, shift: int = 0, wrap: bool = True) -> np.ndarray:
    """The dense [n][n] float64 matrix of the banded A (``env_a`` [band][obs], the device layout)."""
    band = env_a.shape[0]
    half = band // 2
    M = np.zeros((n, n))
    for d in range(band):
        for i in range(n):
            j = i + d - half + shift
            if wrap:
                M[i, j % n] += float(env_a[d, i])
            elif 0 <= j < n:
                M[i, j] += float(env_a[d, i])
    return M


def _weights(table, idx, theta, sigma, sizes, pairs):
    """Per evaluation (pair k, sign s) in order (k0 +, k0 -, k1 +, ...): [(W^T [N, in, out], b [N, out], theta's b)] in
    float64."""
    s = float(np.float32(sigma))
    th = np.asarray(theta, np.float64)
    P = len(th)
    rows = []
    for k in pairs:
        eps = np.asarray(table[int(idx[k]):int(idx[k]) + P], np.float64)
        rows += [th + s * eps, th - s * eps]
    flat = np.stack(rows)
    out, off = [], 0
    for fi, fo in zip(sizes[:-1], sizes[1:]):
        W = flat[:, off:off + fi * fo].reshape(-1, fo, fi)
        out.append((np.ascontiguousarray(W.transpose(0, 2, 1)), flat[:, off + fi * fo:off + fi * fo + fo].copy(),
                    th[off + fi * fo:off + fi * fo + fo]))
        off += fi * fo + fo
    return out


def normalise(ob, mean, std, clip):
    """nn.py:45's ``torch.clamp((ob - mean) / std, -clip, clip)`` in float64: np.clip keeps a NaN and clips +-inf, as
    torch.clamp does."""
    return np.clip((ob - mean) / std, -clip, clip)


def simulate(table, idx, theta, sigma, sizes, ob_mean, ob_std, clip, obs0, env_a, env_b, rew_vec, pos_scale,
             act_noise=None, episodes: int = 1, pairs: Optional[Sequence[int]] = None, variants=(None,), obs0_shift=None,
             activation=np.tanh, fall_height=None, binned=None):
    """The truth (variant None) and its variants for the pairs ``pairs`` (default: all).  ``variants``: mutations (tuples of
    ``mutations``) or None.  ``obs0_shift``: [V][obs] added to obs0 per variant (``growth``).  ``activation``: the policy's
    float64 activation after every layer in place of tanh (f64_rollout's forms), or a list of one per layer; the env's
    own tanh stays.  ``fall_height``: the env's h (None: no episode ends early, a NaN position included).  ``binned``:
    (bins, low, high) of an FFBinned head, whose last layer has act * bins outputs.  ``act_noise``: [n_pairs][2][E T act]
    (or any shape of that size).

    Returns a dict of arrays indexed [V][2][n] ([V][2][n][...] for vectors): float64 'fit', 'mass', 'behv' (3), 'mag' (3),
    'osum', 'osq', 'oabs' (obs: the column sums of ob, ob^2 and |ob|), 'olast' (obs), 'gap' (the smallest | |z_t| - h | over
    the executed steps: a position off by less decides every fall as the truth does; inf without h), 'margin' (a binned
    head's smallest gap between a dimension's two largest outputs over the executed steps; inf without one), 'zmax' (the
    largest |z_t| executed), 'z0' (|z| after the last episode's first step); int64 'steps' (the last episode's t_d), 'used'
    (noise values consumed, sum_e (t_{d,e} + 1) act), 'eps' ([E]: every episode's t_d); and, with ``obs0_shift``, 'dev': the
    largest ||ob_v - ob_0|| over the steps and episodes."""
    idx = np.asarray(idx)
    pairs = list(range(len(idx)) if pairs is None else pairs)
    T, act = rew_vec.shape
    obs, L = sizes[0], len(sizes) - 1
    E = int(episodes)
    V = len(variants)
    N = 2 * len(pairs)
    layers = _weights(table, idx, theta, sigma, sizes, pairs)
    acts = [np.tanh] * L if binned is not None else f64.per_layer(activation, L)
    c = np.asarray(rew_vec, np.float64)
    B = np.asarray(env_b, np.float64)                      # [act][obs]: pre += a @ B
    A = _env_matrix(env_a, obs).T.copy()                   # pre += ob @ A
    mean = np.asarray(ob_mean, np.float64)
    std = np.asarray(ob_std, np.float64)
    ps = float(np.float32(pos_scale))
    h_fall = None if fall_height is None else float(np.float32(fall_height))
    nz_all = None                                          # [N][E T act]: each evaluation's flat run
    if act_noise is not None:
        nz_all = np.asarray(act_noise, np.float32).reshape(len(idx), 2, -1)[pairs].reshape(N, -1).astype(np.float64)

    # per-variant parameters
    def flag(name):
        return np.array([v is not None and v[0] == name for v in variants])

    act_mask = [np.ones((V, d)) for d in sizes[1:]]
    in_mask = [np.ones((V, d)) for d in sizes[:-1]]
    stale = [np.zeros(V, bool) for _ in range(L)]
    unpert = [np.zeros(V, bool) for _ in range(L)]
    for v, m in enumerate(variants):
        if m is None:
            continue
        if m[0] == 'row':
            act_mask[m[1]][v, m[2]] = 0.0
        elif m[0] == 'col':
            in_mask[m[1]][v, m[2]] = 0.0
        elif m[0] == 'stale':
            stale[m[1]][v] = True
        elif m[0] == 'bias':
            unpert[m[1]][v] = True
    alt_A = [(v, _env_matrix(env_a, obs, shift=1).T.copy() if m[0] == 'band_shift' else _env_matrix(env_a, obs, wrap=False).T.copy())
             for v, m in enumerate(variants) if m is not None and m[0] in ('band_shift', 'band_nowrap')]
    b_last = flag('b_last_col')
    vmean = np.where(flag('no_mean')[:, None], 0.0, mean[None, :])            # [V][obs]
    vclip = np.where(flag('no_clip'), np.inf, float(clip))[None, :, None]     # [1][V][1]
    tfac = np.where(flag('tanh_approx'), 1.0 + TANH_APPROX, 1.0)[None, :, None]
    drop_last, skip_first = flag('drop_last_step'), flag('skip_first_env_step')
    env_clean, rew_clean = flag('env_clean'), flag('rew_clean')
    no_reset_obs, no_reset_pos, first_out = flag('no_reset_obs'), flag('no_reset_pos'), flag('first_episode_outputs')
    ep0_noise = flag('ep0_noise')[None, :]                                     # [1][V]
    ev_src = np.where(flag('swap_sign_noise')[None, :], (np.arange(N) ^ 1)[:, None], np.arange(N)[:, None])  # [N][V]
    any_masks = [not np.all(m == 1.0) for m in act_mask], [not np.all(m == 1.0) for m in in_mask]
    o0 = np.broadcast_to(np.asarray(obs0, np.float64), (N, V, obs)).copy()
    if obs0_shift is not None:
        o0 += np.asarray(obs0_shift, np.float64)[None, :, :]
    # bias per (evaluation, variant)
    biases = [np.where(unpert[l][None, :, None], th_b[None, None, :], b[:, None, :]) for l, (_, b, th_b) in enumerate(layers)]

    fit, mass = np.zeros((N, V)), np.zeros((N, V))
    res = {}
    ob = o0.copy()
    pos = np.zeros((N, V, 3))
    prev = [np.zeros((N, V, d)) for d in sizes[1:]]
    dev = np.zeros((N, V))
    cols = [0, 1 % act, 2 % act]
    used = np.zeros((N, V), np.int64)
    eps = np.zeros((N, V, E), np.int64)
    gap, margin = np.full((N, V), np.inf), np.full((N, V), np.inf)
    zmax, z0 = np.zeros((N, V)), np.zeros((N, V))
    for e in range(E):
        ob = np.where(no_reset_obs[None, :, None] & (e > 0), ob, o0)
        pos = np.where(no_reset_pos[None, :, None] & (e > 0), pos, 0.0)
        mag = np.zeros((N, V, 3))
        osum, osq, oabs = (np.zeros((N, V, obs)) for _ in range(3))
        alive = np.ones((N, V), bool)
        t_d = np.full((N, V), T - 1, np.int64)
        start = np.where(ep0_noise, 0, used)                                     # [N][V]: this episode's noise offset
        for t in range(T):
            if not alive.any():
                break
            run = alive & ~(drop_last & (t == T - 1))                           # [N][V]: the step is taken
            h = normalise(ob, vmean[None], std, vclip)
            for l, (WT, _, _) in enumerate(layers):
                if any_masks[1][l]:
                    h = h * in_mask[l][None]
                z = np.matmul(h, WT) + biases[l]
                y = acts[l](z) * tfac
                if any_masks[0][l]:
                    y = y * act_mask[l][None]
                if l + 1 < L and stale[l + 1].any():
                    nxt = np.where(stale[l + 1][None, :, None], prev[l], y)
                    prev[l] = y
                    h = nxt
                else:
                    h = y
            if binned is not None:
                bins, low, high = binned
                out = h.reshape(N, V, act, bins)
                top = np.sort(out, axis=3)
                margin = np.where(alive, np.minimum(margin, (top[..., -1] - top[..., -2]).min(axis=2)), margin)
                lo = np.asarray(low, np.float64)
                a = lo + (np.asarray(high, np.float64) - lo) * out.argmax(axis=3) / (bins - 1.0)
            else:
                a = h                                                           # [N][V][act]
            if nz_all is not None:
                nz = nz_all[ev_src[:, :, None], start[:, :, None] + t * act + np.arange(act)]    # [N][V][act]
                if binned is None and any_masks[0][L - 1]:
                    nz = nz * act_mask[L - 1][None]                              # a row never written gets no noise either
                an = a + nz
                a_env = np.where(env_clean[None, :, None], a, an)
                a_rew = np.where(rew_clean[None, :, None], a, an)
            else:
                a_env = a_rew = a
            prod = a_rew * c[t]
            fit += np.where(run, prod.sum(axis=2), 0.0) / E
            mass += np.where(run, np.abs(prod).sum(axis=2), 0.0) / E
            term = ps * a_rew[:, :, cols] * run[:, :, None]
            npos = pos + term
            lv = alive[:, :, None]
            mag = np.where(lv, mag + (np.abs(npos) + np.abs(term)), mag)
            pos = np.where(lv, npos, pos)
            pre = ob @ A
            for v, Av in alt_A:
                pre[:, v] = ob[:, v] @ Av
            pre += a_env @ B
            if b_last.any():
                pre[:, b_last] -= a_env[:, b_last, -1:] * B[-1][None, None, :]
            nob = np.tanh(pre) * tfac
            if t == 0:
                nob = np.where(skip_first[None, :, None], ob, nob)
            rv = run[:, :, None]
            ob = np.where(rv, nob, ob)
            if obs0_shift is not None:
                dev = np.maximum(dev, np.sqrt(((ob - ob[:, :1]) ** 2).sum(axis=2)))
            osum += ob * rv
            osq += ob * ob * rv
            oabs += np.abs(ob) * rv
            zt = np.abs(pos[:, :, 2])
            if t == 0:
                z0 = zt
            zmax = np.where(alive, np.maximum(zmax, zt), zmax)
            fell = False
            if h_fall is not None:
                gap = np.where(alive, np.minimum(gap, np.abs(zt - h_fall)), gap)
                fell = ~(zt <= h_fall)
            ended = alive & (fell | (t == T - 1))
            t_d[ended] = t
            alive &= ~ended
        eps[:, :, e] = t_d
        used += (t_d + 1) * act
        out = dict(behv=pos.copy(), mag=mag, osum=osum, osq=osq, oabs=oabs, olast=ob.copy())
        if e == 0:
            first = out
        if e == E - 1:
            for k, val in out.items():
                res[k] = np.where(first_out.reshape((1, V) + (1,) * (val.ndim - 2)), first[k], val)
    res.update(fit=fit, mass=mass, steps=t_d, used=used, eps=eps, gap=gap, margin=margin, zmax=zmax, z0=z0)
    if obs0_shift is not None:
        res['dev'] = dev

    def shape(x):  # [N][V][...] -> [V][2][n][...]
        x = np.moveaxis(x, 1, 0)
        return x.reshape((V, len(pairs), 2) + x.shape[2:]).swapaxes(1, 2)
    return {k: shape(v) for k, v in res.items()}


def truth(*args, **kw):
    """The unmutated truth: ``simulate`` with one variant, the [V] axis dropped."""
    kw.pop('variants', None)
    return {k: v[0] for k, v in simulate(*args, variants=(None,), **kw).items()}


def growth(*args, directions: int = 3, delta: float = 1e-9, seed: int = 0, **kw):
    """The largest ||dob_t|| / ||dob_0|| over the steps and episodes (and the evaluations) for obs0 moved by ``delta`` along a
    few random directions: how far the loop carries a rounding difference.  ``kw`` as ``simulate`` takes them (activation,
    fall_height, binned, ...)."""
    obs = args[4][0]                                                           # sizes[0]
    rs = np.random.RandomState(seed)
    d = rs.randn(directions, obs)
    d *= delta / np.linalg.norm(d, axis=1, keepdims=True)
    shift = np.concatenate([np.zeros((1, obs)), d])
    r = simulate(*args, variants=(None,) * (directions + 1), obs0_shift=shift, **kw)
    return float(r['dev'][1:].max() / delta)
