"""Both closed-loop kernels against the float64 truth (tests/closed_f64.py): rollout_closed.cu (one CTA per pair) and
rollout_closedw.cu (one thread-block cluster per evaluation), noise-free and with action noise and episodes, at the shipped
configs' policies and at the launch and layout edges.

The problems (``PROBLEMS``) come in two regimes: ``init``, weights and biases of scale g / sqrt(fan_in) with g = 1 (near
torch's default initialisation), and ``sat``, g = 2 or 3, where actions are O(1) and the tanh layers saturate.  Each one was
chosen on the CPU (tests/test_closed_f64_host.py) so that a 1e-9 move of the start observation grows at most 100-fold over the
episode: the loop does not amplify rounding, so a float32 kernel stays within rounding of the truth, and the same file shows
that every modelled kernel bug (closed_f64.MUTATIONS: a missing row, a skipped column, a stale activation buffer, a wrong band
index, misplaced noise, episodes not reset, ...) moves a checked value by at least 10 times its bound on some problem of
every shape.

One assert helper (``_check``) judges every case:
* per evaluation ``|f - truth| <= EVAL_REL * mass`` (the open-loop float32 bound, mass = sum_t mean_e sum_j |a_tj c_tj|);
* over the evaluations ``rms(f - truth) <= RMS_BOUND * spread`` (spread = the truth's standard deviation, floored at
  1e-3 sqrt(T));
* final positions within ``2 * 2^-24 * mag + ACT_ERR * pos_scale * T`` (float32 rounding of the T-term sums, plus the actions'
  own error);
* the ObStat sums of the saved evaluations within T ulps of their magnitude per saved evaluation plus ``OBS_ERR`` per
  observation; the ObStat count exact.
Largest values measured on an H100 SXM (80 GB) over this file: max err/mass 3.1e-6 (obj-sat; the init
regime stays below 1.5e-6), rms/spread 1.55e-4 (cta17_noise0.05_E1-sat, 40 steps: a small spread).  The saturating regime
sits well above the float32 oracle (<= 8.6e-7 of the mass on the CPU) because both kernels use a fast tanh with an absolute
error of ~1e-7, which a weight scale of g = 3 amplifies through every layer; RMS_BOUND is about 2x the measured maximum.

Which kernel and cluster size a case takes is restated (closed_f64.plan) and asserted through ``Engine.closed_mlp_plan``, and
every case is one launch (``Engine.launches``), so a dispatch change fails here instead of silently moving a case.
"""
import math
import os
import sys
from typing import NamedTuple, Tuple

import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closed_f64 as cf  # noqa: E402
from closed_f64 import ACT_ERR, EVAL_REL, OBS_ERR, RMS_BOUND, U  # noqa: E402

pytestmark = pytest.mark.gpu

SIGMA = 0.02


class Problem(NamedTuple):
    name: str
    sizes: Tuple[int, ...]
    T: int
    g: float                    # weight scale g / sqrt(fan_in)
    b_gain: float               # ClosedLoopEnvSpec.b_gain: how strongly the actions drive the env
    seed: int
    band: int = 8
    n_pairs: int = 3
    E: int = 1
    ac_std: float = 0.0
    fit_stride: int = 1

    @property
    def regime(self):
        return 'init' if self.g == 1 else 'sat'

    @property
    def id(self):
        return f'{self.name}-{self.regime}'


def largest_eight_cta_width():
    """The family 384-256-256-h-64 (band 16): the largest h whose cluster still fits 8 CTAs (restated plan)."""
    return max(h for h in range(1, 257) if cf.cluster_size([384, 256, 256, h, 64], 16) is not None)


def _shapes():
    H8 = largest_eight_cta_width()
    return [  # name, sizes, T, extra
        ('simple_conf', (15, 256, 256, 3), 300, dict(fit_stride=2)),
        ('obj', (17, 256, 256, 256, 6), 300, {}),
        ('obj26', (26, 256, 256, 256, 6), 300, {}),
        ('obj28', (28, 256, 256, 256, 8), 300, {}),
        ('flagrun', (28, 128, 256, 256, 128, 8), 300, dict(E=10, ac_std=0.01)),
        ('ns', (28, 256, 256, 256, 8), 10_000, dict(n_pairs=2)),
        ('humanoid_wide', (376, 256, 256, 17), 200, {}),
        ('cta376', (376, 64, 64, 17), 200, {}),
        ('cta17', (17, 64, 64, 6), 300, {}),
        ('width1_65', (20, 1, 65, 5), 60, {}),
        ('act1', (20, 96, 80, 1), 60, {}),
        ('act64', (20, 130, 70, 64), 60, {}),
        ('obs_eq_band', (8, 100, 100, 4), 60, {}),
        ('obs384_band16', (384, 128, 128, 8), 40, dict(band=16)),
        ('T1', (15, 256, 256, 3), 1, {}),
        ('T2', (15, 256, 256, 3), 2, {}),
        ('eight_ctas', (384, 256, 256, H8, 64), 12, dict(band=16, n_pairs=2)),
    ]


# the saturating regime's (g, b_gain, seed) per shape: picked on the CPU among g = 2, 3 and b_gain 0.1 .. 0.5 for a growth well
# below 100 (test_closed_f64_host.py prints it); the same shape at a larger b_gain or g is often chaotic (growth ~1e9)
_SAT = {'simple_conf': (3.0, 0.5, 3), 'T1': (3.0, 0.5, 3), 'T2': (3.0, 0.5, 3), 'obj': (3.0, 0.1, 4), 'obj26': (3.0, 0.1, 4),
        'obj28': (2.0, 0.1, 3), 'ns': (2.0, 0.1, 4), 'flagrun': (2.0, 0.1, 3), 'humanoid_wide': (3.0, 0.1, 4),
        'cta376': (2.0, 0.3, 3), 'cta17': (3.0, 0.2, 4), 'width1_65': (3.0, 0.2, 4), 'act1': (3.0, 0.1, 4),
        'act64': (3.0, 0.1, 4), 'obs_eq_band': (3.0, 0.2, 4), 'obs384_band16': (3.0, 0.1, 4), 'eight_ctas': (2.0, 0.2, 3)}
_NOISE = [('cta17', (17, 64, 64, 6)), ('simple_conf', (15, 256, 256, 3)), ('flagrun', (28, 128, 256, 256, 128, 8))]


def _problems():
    out = []
    for name, sizes, T, extra in _shapes():
        out.append(Problem(name, sizes, T, 1.0, 0.5, 3, **extra))
        out.append(Problem(name, sizes, T, *_SAT[name], **extra))
    for name, sizes in _NOISE:
        for ac_std in (0.01, 0.05):
            for E in (1, 2, 10):
                nm = f'{name}_noise{ac_std}_E{E}'
                out.append(Problem(nm, sizes, 40, 1.0, 0.5, 5, E=E, ac_std=ac_std))
                out.append(Problem(nm, sizes, 40, *_SAT[name], E=E, ac_std=ac_std))
    return out


PROBLEMS = _problems()
# a problem that amplifies rounding (the calibration must refuse it): 17-256^3-6 at g = 2, b_gain 0.5
CHAOTIC = Problem('obj_chaotic', (17, 256, 256, 256, 6), 300, 2.0, 0.5, 3)


def build(p: Problem):
    """The host inputs of a problem: a dict of everything the kernels and the truth take."""
    sizes = list(p.sizes)
    P = orc.n_params(orc.layer_dims(sizes[0], sizes[1:-1], sizes[-1]))
    rs = np.random.RandomState(p.seed)
    table = rs.randn(P + 50_000).astype(np.float32)
    parts = []
    for fi, fo in zip(sizes[:-1], sizes[1:]):
        parts.append(rs.randn(fi * fo + fo) * (p.g / math.sqrt(fi)))
    theta = np.concatenate(parts).astype(np.float32)
    idx = rs.randint(0, len(table) - P, size=p.n_pairs).astype(np.int64)
    spec = orc.ClosedLoopEnvSpec(sizes[0], sizes[-1], p.T, band=p.band, b_gain=p.b_gain)
    nr = np.random.RandomState(p.seed + 1)
    mean, std, clip = nr.randn(sizes[0]) * 0.05, 0.5 + nr.rand(sizes[0]), 1.0
    noise = None
    if p.ac_std:
        noise = (np.random.RandomState(p.seed + 2).randn(p.n_pairs, 2, p.E, p.T, sizes[-1]) * p.ac_std).astype(np.float32)
    saved = [(k, s) for k in range(p.n_pairs) for s in range(2) if (k + s) % 2 == 0]
    return dict(sizes=sizes, P=P, table=table, theta=theta, idx=idx, spec=spec, mean=mean, std=std, clip=clip, noise=noise,
                saved=saved, obs0=spec.obs_stream[0].copy(), env_a=np.ascontiguousarray(spec.env_a.T),
                env_b=np.ascontiguousarray(spec.env_b.T))


def truth_args(p: Problem, d):
    """The positional and keyword arguments of closed_f64.simulate / truth / growth for problem ``p``."""
    return ((d['table'], d['idx'], d['theta'], SIGMA, d['sizes'], d['mean'], d['std'], d['clip'], d['obs0'], d['env_a'],
             d['env_b'], d['spec'].rew_vec, d['spec'].pos_scale), dict(act_noise=d['noise'], episodes=p.E))


def saved_mask(p: Problem, saved):
    m = np.zeros((2, p.n_pairs), bool)
    for k, s in saved:
        m[s, k] = True
    return m


def bounds(p: Problem, tr, saved, pos_scale):
    """The per-value bounds ``_check`` applies to the truth ``tr`` (closed_f64.truth's dict): fitness [2][n], position
    [2][n][3], ObStat sum and sum of squares [obs]."""
    m = saved_mask(p, saved)
    ps = float(np.float32(pos_scale))
    ns = max(1, int(m.sum()))
    return dict(fit=EVAL_REL * tr['mass'],
                pos=2 * U * tr['mag'] + ACT_ERR * ps * p.T,
                osum=2 * p.T * U * tr['oabs'][m].sum(axis=0) + OBS_ERR * p.T * ns,
                osq=2 * p.T * U * tr['osq'][m].sum(axis=0) + 2 * OBS_ERR * p.T * ns)


def coins(n, saved):
    c = np.full((n, 4), 0xFFFFFFFF, dtype=np.uint32)
    for k, sgn in saved:
        c[k, 2 * sgn:2 * sgn + 2] = 0                                               # u = 0 < chance
    return c


# ---------------------------------------------------------------------------------------------- the device
def _run(eng, p: Problem, d):
    """One rollout_closed_mlp call: (fitness [2][n], behaviour [2][n][3], ObStat sum, sumsq, count, launches)."""
    n, obs, T = p.n_pairs, p.sizes[0], p.T
    fit = torch.full((2, n * p.fit_stride), float('nan'), dtype=torch.float64, device=eng.device)
    behv = torch.full((2, n, 3), float('nan'), dtype=torch.float32, device=eng.device)
    osum, osq = (torch.zeros(obs, dtype=torch.float64, device=eng.device) for _ in range(2))
    ocnt = torch.zeros(2, dtype=torch.float64, device=eng.device)
    dv = eng.to_device
    spec = d['spec']
    noise = None if d['noise'] is None else dv(np.ascontiguousarray(d['noise']))
    l0 = eng.launches
    eng.rollout_closed_mlp(dv(d['table']), dv(d['idx']), dv(d['theta']), SIGMA, list(p.sizes), dv(d['mean']), dv(d['std']),
                           d['clip'], dv(d['obs0']), dv(d['env_a']), dv(d['env_b']), dv(spec.rew_vec), spec.pos_scale, fit[0],
                           fit[1], p.fit_stride, behv[0].view(-1), behv[1].view(-1),
                           coin_words=dv(coins(n, d['saved']).view(np.int32)), save_obs_chance=0.5, ob_sum=osum, ob_sumsq=osq,
                           ob_count=ocnt, act_noise=noise, episodes=p.E)
    eng.sync()
    launches = eng.launches - l0
    f = fit.cpu().numpy()
    if p.fit_stride > 1:                                     # the other objective's column is untouched
        assert np.isnan(f.reshape(2, n, p.fit_stride)[:, :, 1:]).all()
    f = f[:, ::p.fit_stride]
    b = behv.cpu().numpy()
    assert not np.isnan(f).any() and not np.isnan(b).any(), 'an evaluation was not written'
    return f, b, osum.cpu().numpy(), osq.cpu().numpy(), ocnt.cpu().numpy(), launches


def _check(tag, p: Problem, got, tr, saved, pos_scale):
    """The one assert helper.  ``got``: _run's first five values; ``tr``: the truth."""
    f, b, osum, osq, ocnt = got
    bd = bounds(p, tr, saved, pos_scale)
    m = saved_mask(p, saved)
    err = np.abs(f - tr['fit'])
    spread = max(tr['fit'].std(), 1e-3 * math.sqrt(p.T))
    rms = math.sqrt((err ** 2).mean())
    worst = (err / tr['mass']).max()
    print(f'\n[closed f64] {tag}: max err/mass {worst:.3g} (bound {EVAL_REL:.3g}), rms/spread {rms / spread:.3g} '
          f'(bound {RMS_BOUND:.3g})')
    assert np.all(err <= bd['fit']), (tag, worst)
    assert rms <= RMS_BOUND * spread, (tag, rms / spread)
    assert np.all(np.abs(b - tr['behv']) <= bd['pos']), (tag, np.abs(b - tr['behv']).max())
    assert np.all(np.abs(osum - tr['osum'][m].sum(axis=0)) <= bd['osum']), tag
    assert np.all(np.abs(osq - tr['osq'][m].sum(axis=0)) <= bd['osq']), tag
    assert ocnt.tolist() == [float(len(saved) * p.T), float(len(saved))], tag


@pytest.mark.parametrize('p', PROBLEMS, ids=[p.id for p in PROBLEMS])
def test_closed_kernels_match_the_float64_truth(eng, p):
    d = build(p)
    C = cf.plan(p.sizes, p.band)
    assert eng.closed_mlp_plan(list(p.sizes), p.band)[0] == C
    got = _run(eng, p, d)
    assert got[5] == 1
    args, kw = truth_args(p, d)
    _check(f'{p.id} C={C}', p, got[:5], cf.truth(*args, **kw), d['saved'], d['spec'].pos_scale)


# ---------------------------------------------------------------------------------------------- a NaN in the observation mean
# torch.clamp (nn.py:45) keeps a NaN, so a NaN in ob_mean makes that observation column NaN at every step: every output of a
# tanh or activation stack and every fitness is NaN, in the float64 truth and on the device.  A binned head's arg-max over
# all-NaN outputs is bin 0 (torch.argmax), so its fitness stays finite and is held to the binned tests' bound.  On the
# cluster kernel (the closed loop's wide and activation families) the position is NaN too, and an env without a fall height
# still runs every saved evaluation's T steps: ob_count is [T saved, saved].
_NAN_FAMILIES = [('one_cta', (17, 64, 64, 6), None, 0), ('wide', (15, 256, 256, 3), None, 0),
                 ('activation', (17, 64, 64, 6), 'relu', 0), ('binned', (15, 64, 64, 15), None, 5)]


@pytest.mark.parametrize('loop', ['open', 'closed'])
@pytest.mark.parametrize('name,sizes,act_kind,bins', _NAN_FAMILIES, ids=[f[0] for f in _NAN_FAMILIES])
def test_nan_in_the_observation_mean_reaches_the_fitness(eng, name, sizes, act_kind, bins, loop):
    import f64_rollout as f64
    from es_pytorch_b200 import _lib
    from es_pytorch_b200.nn.nn import Activation, BinnedHead
    sizes, T, n = list(sizes), 30, 3
    obs = sizes[0]
    adim = sizes[-1] // bins if bins else sizes[-1]
    head = BinnedHead(bins, np.float32([-1.0, 0.0, 0.5]), np.float32([1.0, 2.0, 0.75])) if bins else None
    activation = Activation(_lib.ES_ACT_RELU, 0.0) if act_kind else None
    f64_act = f64.relu if act_kind else np.tanh
    P = orc.n_params(orc.layer_dims(obs, sizes[1:-1], sizes[-1]))
    rs = np.random.RandomState(len(sizes) + obs)
    table, theta = rs.randn(P + 20_000).astype(np.float32), (rs.randn(P) * 0.1).astype(np.float32)
    idx = rs.randint(0, 20_000, size=n).astype(np.int64)
    mean, std, clip = rs.randn(obs) * 0.05, 0.5 + rs.rand(obs), 1.0
    mean[1] = np.nan
    dv = eng.to_device
    spec = orc.ClosedLoopEnvSpec(obs, adim, T, band=8) if loop == 'closed' else orc.SyntheticEnvSpec(obs, adim, T)
    fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
    ob, saved = {}, []
    if loop == 'closed' and name in ('wide', 'activation'):
        saved = [(s, k) for s in range(2) for k in range(n) if (k + s) % 2 == 0]
        coins = np.full((n, 4), 0xFFFFFFFF, dtype=np.uint32)
        for s, k in saved:
            coins[k, 2 * s:2 * s + 2] = 0                                       # u = 0 < chance
        ob = dict(coin_words=dv(coins.view(np.int32)), save_obs_chance=0.5,
                  ob_sum=torch.zeros(obs, dtype=torch.float64, device=eng.device),
                  ob_sumsq=torch.zeros(obs, dtype=torch.float64, device=eng.device),
                  ob_count=torch.zeros(2, dtype=torch.float64, device=eng.device))
    if loop == 'open':
        obsn = eng.normalise_obs(dv(spec.obs_stream[:T]), dv(mean), dv(std), clip)
        eng.rollout(dv(table), dv(idx), dv(theta), SIGMA, sizes, obsn, dv(spec.rew_vec[:T]), spec.pos_scale, fit[0], fit[1], 1,
                    behv[0], behv[1], head=head, activation=activation)
    else:
        eng.rollout_closed_mlp(dv(table), dv(idx), dv(theta), SIGMA, sizes, dv(mean), dv(std), clip, dv(spec.obs_stream[0].copy()),
                               dv(np.ascontiguousarray(spec.env_a.T)), dv(np.ascontiguousarray(spec.env_b.T)), dv(spec.rew_vec),
                               spec.pos_scale, fit[0], fit[1], 1, behv[0].view(-1), behv[1].view(-1), head=head,
                               activation=activation, **ob)
    eng.sync()
    f = fit.cpu().numpy()
    if ob:
        assert ob['ob_count'].cpu().tolist() == [float(T * len(saved)), float(len(saved))]
    if bins:                                   # the oracle's per-step loop: torch.argmax of the NaN outputs
        dims = orc.layer_dims(obs, sizes[1:-1], sizes[-1])
        want, bound = np.zeros((2, n)), np.zeros((2, n))
        for k, i in enumerate(idx):
            for s, sign in enumerate((1.0, -1.0)):
                layers = orc.unflatten(orc.pheno_params(theta, SIGMA, sign * orc.table_get(table, int(i), P)), dims)
                rews = orc.run_model(spec, layers, mean, std, clip, T, binned=(bins, head.low, head.high))[0]
                want[s, k], bound[s, k] = sum(rews), 2e-5 * max(1.0, np.abs(rews).sum())
        assert np.isfinite(want).all()
    elif loop == 'open':
        obsn_h = orc.normalise_obs(spec.obs_stream[:T], mean, std, clip)
        want, _, mass, _ = f64.rollout_f64(table, idx, theta, SIGMA, sizes, obsn_h, spec.rew_vec[:T], spec.pos_scale,
                                           activation=f64_act)
        bound = EVAL_REL * mass
        assert np.isnan(want).all()
    else:
        tr = cf.truth(table, idx, theta, SIGMA, sizes, mean, std, clip, spec.obs_stream[0], spec.env_a.T, spec.env_b.T,
                      spec.rew_vec, spec.pos_scale, activation=f64_act)
        want, bound = tr['fit'], EVAL_REL * tr['mass']
        assert np.isnan(want).all()
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(f), nan), f
    assert np.all(np.abs(f[~nan] - want[~nan]) <= bound[~nan]), (f, want)
