"""CPU calibration of every problem of tests/test_gpu_closed_f64.py against the float64 truth (tests/closed_f64.py).

For every problem:
(a) the loop does not amplify rounding: a 1e-9 move of the start observation grows at most 100-fold over the episode
    (closed_f64.growth); a known-chaotic problem is refused by the same gate;
(b) the float32 oracle (es_oracle.run_model, fed the problem's noise array) is within 1e-6 of the reward
    mass of the truth for every evaluation: a tenth of the GPU bound, so the bound has room for a float32 kernel;
(c) with sigma = 0 the truth's two signs are identical and match the float32 oracle to float32 grade (the truth itself);
(d) for each kernel and each shape, every modelled bug (closed_f64.mutations) moves the fitness, a position or an ObStat sum by
    at least 10 times the GPU test's bound on at least one of that shape's problems, so a kernel with that bug fails there.
Each problem prints its growth, its float32-oracle error over the mass and its weakest mutation ratio.
"""
import os
import sys
from collections import defaultdict

import numpy as np
import pytest

from oracle import es_oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closed_f64 as cf  # noqa: E402
import test_gpu_closed_f64 as G  # noqa: E402

GROWTH_MAX = 100.0
ORACLE_REL = 1e-6
MUT_MIN = 10.0
# problems whose mutation runs would take minutes (ns: T = 10 000); their shape is covered by a shorter problem (obj28)
_MUT_SKIP = {'ns'}


class _Stream:
    """A RandomState stand-in whose randn returns the next values of a fixed gaussian array (the problem's noise / ac_std)."""

    def __init__(self, flat):
        self.flat, self.at = flat, 0

    def randn(self, m):
        v = self.flat[self.at:self.at + m]
        self.at += m
        return v


def _oracle(p, d, k, s, sigma=G.SIGMA):
    dims = orc.layer_dims(p.sizes[0], p.sizes[1:-1], p.sizes[-1])
    sign = 1.0 if s == 0 else -1.0
    layers = orc.unflatten(orc.pheno_params(d['theta'], sigma, sign * orc.table_get(d['table'], int(d['idx'][k]), d['P'])), dims)
    if d['noise'] is None:
        return orc.run_model(d['spec'], layers, d['mean'], d['std'], d['clip'], p.T)
    rs = _Stream(d['noise'][k, s].reshape(-1).astype(np.float64) / p.ac_std)
    return orc.run_model(d['spec'], layers, d['mean'], d['std'], d['clip'], p.T, ac_std=p.ac_std, rs=rs, episodes=p.E)


_cache = {}


def _truth(p):
    if p not in _cache:
        d = G.build(p)
        args, kw = G.truth_args(p, d)
        _cache.clear()
        _cache[p] = d, args, kw, cf.truth(*args, **kw)
    return _cache[p]


def mutation_ratios(p):
    """{mutation: the largest |mutated - truth| / bound over the checked values} for problem ``p``."""
    d, args, kw, tr = _truth(p)
    muts = cf.mutations(p.sizes, p.band, p.ac_std != 0, p.E)
    r = cf.simulate(*args, variants=[None] + muts, **kw)
    m = G.saved_mask(p, d['saved'])
    bd = G.bounds(p, tr, d['saved'], d['spec'].pos_scale)
    out = {}
    for v, mu in enumerate(muts, start=1):
        ratios = [np.max(np.abs(r['fit'][v] - r['fit'][0]) / bd['fit']),
                  np.max(np.abs(r['behv'][v] - r['behv'][0]) / bd['pos']),
                  np.max(np.abs(r['osum'][v][m].sum(axis=0) - r['osum'][0][m].sum(axis=0)) / bd['osum']),
                  np.max(np.abs(r['osq'][v][m].sum(axis=0) - r['osq'][0][m].sum(axis=0)) / bd['osq'])]
        out[mu] = float(max(ratios))
    return out


def _kernel(p):
    return 'one-CTA' if cf.plan(p.sizes, p.band) == 0 else 'cluster'


@pytest.mark.parametrize('p', G.PROBLEMS, ids=[p.id for p in G.PROBLEMS])
def test_problem_is_stable_and_the_oracle_is_within_a_tenth_of_the_bound(p):
    d, args, kw, tr = _truth(p)
    gr = cf.growth(*args, **kw)
    worst = 0.0
    for k in range(p.n_pairs):
        for s in range(2):
            rews, bh, _, _ = _oracle(p, d, k, s)
            worst = max(worst, abs(sum(rews) - tr['fit'][s, k]) / tr['mass'][s, k])
    print(f'\n[closed f64 host] {p.id}: growth {gr:.3g}, float32 oracle err/mass {worst:.3g}')
    assert gr <= GROWTH_MAX, (p.id, gr)
    assert worst <= ORACLE_REL, (p.id, worst)


def test_a_chaotic_problem_is_refused():
    p = G.CHAOTIC
    d = G.build(p)
    args, kw = G.truth_args(p, d)
    gr = cf.growth(*args, **kw)
    print(f'\n[closed f64 host] {p.id}: growth {gr:.3g}')
    assert gr > 1e3 * GROWTH_MAX


_SIGMA0 = [p for p in G.PROBLEMS if p.regime == 'init' and p.T <= 300 and p.name not in _MUT_SKIP]


@pytest.mark.parametrize('p', _SIGMA0, ids=[p.id for p in _SIGMA0])
def test_truth_at_sigma_zero_matches_the_float32_oracle(p):
    d = G.build(p)
    if d['noise'] is not None:                       # both signs with the + evaluation's noise
        d['noise'][:, 1] = d['noise'][:, 0]
    args, kw = G.truth_args(p, d)
    args = args[:3] + (0.0,) + args[4:]
    tr = cf.truth(*args, pairs=[0], **kw)
    assert np.array_equal(tr['fit'][0], tr['fit'][1]) and np.array_equal(tr['behv'][0], tr['behv'][1])
    rews, bh, ob, _ = _oracle(p, d, 0, 0, sigma=0.0)
    assert abs(sum(rews) - tr['fit'][0, 0]) <= 1e-6 * tr['mass'][0, 0]
    assert np.abs(np.array(bh[-3:]) - tr['behv'][0, 0]).max() <= 2 * cf.U * tr['mag'][0, 0].max() + 1e-7 * p.T
    assert np.abs(ob.astype(np.float64).sum(axis=0) - tr['osum'][0, 0]).max() <= cf.OBS_ERR * p.T


def _groups():
    g = defaultdict(list)
    for p in G.PROBLEMS:
        if p.name not in _MUT_SKIP:
            g[(_kernel(p), p.sizes)].append(p)
    return g


_GROUPS = _groups()


@pytest.mark.parametrize('key', list(_GROUPS), ids=[f'{k}-{"-".join(map(str, s))}' for k, s in _GROUPS])
def test_every_mutation_fails_some_problem_of_each_shape(key):
    best = defaultdict(float)
    for p in _GROUPS[key]:
        rat = mutation_ratios(p)
        weakest = min(rat, key=rat.get)
        print(f'\n[closed f64 host] {p.id}: weakest mutation {weakest} {rat[weakest]:.3g}x')
        for mu, r in rat.items():
            best[mu] = max(best[mu], r)
    missed = {mu: r for mu, r in best.items() if r < MUT_MIN}
    assert not missed, (key, missed)


def test_the_observation_clip_is_torch_clamp():
    """The oracle's normalise_obs and the float64 truth's clip (closed_f64.normalise) against torch.clamp
    (nn.py:45): a NaN stays NaN, +-inf becomes +-clip, +-clip and the values next to it are exact.  The GPU tests of a NaN
    in the observation mean compare against these."""
    import torch
    clip = 5.0
    x = np.array([np.nan, np.inf, -np.inf, clip, -clip, np.nextafter(clip, 9), np.nextafter(-clip, -9), np.nextafter(clip, 0),
                  0.0, -0.0, 1e30, -1e-30])
    want = torch.clamp(torch.from_numpy(x), -clip, clip).numpy()
    assert np.isnan(want[0]) and list(want[1:5]) == [clip, -clip, clip, -clip]
    got = cf.normalise(x, np.zeros_like(x), np.ones_like(x), clip)
    assert np.array_equal(got, want, equal_nan=True) and np.array_equal(np.signbit(got), np.signbit(want))
    ob = x.astype(np.float32)
    got32 = orc.normalise_obs(ob, np.zeros_like(x), np.ones_like(x), clip)
    want32 = torch.clamp(torch.from_numpy(ob).double(), -clip, clip).float().numpy()
    assert np.array_equal(got32, want32, equal_nan=True)
    # a NaN in the mean, and an infinite one, through the closed-loop truth: every fitness NaN / every fitness finite
    sizes, T = [4, 3, 2], 3
    P = orc.n_params(orc.layer_dims(4, [3], 2))
    rs = np.random.RandomState(0)
    table, theta, idx = rs.randn(P + 10).astype(np.float32), rs.randn(P).astype(np.float32), np.array([0, 5])
    spec = orc.ClosedLoopEnvSpec(4, 2, T, band=2)
    for m, finite in (([np.nan, 0, 0, 0], False), ([np.inf, -np.inf, 0, 0], True)):
        args = (table, idx, theta, 0.02, sizes, np.array(m), np.ones(4), clip, spec.obs_stream[0], spec.env_a.T, spec.env_b.T,
                spec.rew_vec, spec.pos_scale)
        f = cf.truth(*args)['fit']
        assert (np.isfinite(f) if finite else np.isnan(f)).all(), f
