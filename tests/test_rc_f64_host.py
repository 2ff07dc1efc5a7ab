"""CPU calibration of tests/test_gpu_reconstruct_f64.py's problems against the float64 truth (tests/rc_f64.py).

On a sample of each problem's columns (the lane, warp and tile edges, the last tile and a random spread):
(a) the kernel's summation order, emulated in float32 (rc_f64.emulate), passes both checks of rc_f64.judge;
(b) for each group of problems, every modelled kernel bug (rc_f64.MUTATIONS) that can occur in the group exceeds one of the checks
    at least tenfold on some problem of the group, so a kernel with that bug fails there.
Each group prints every mutation's best margin; the weakest is the number that matters.
"""
import os
import sys
from collections import defaultdict

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rc_f64 as rc  # noqa: E402
import test_gpu_reconstruct_f64 as G  # noqa: E402

MUT_MIN = 10.0


def sample_cols(P: int, seed: int) -> np.ndarray:
    """Columns 0-40 and 90-140 (lanes and warps), +-3 around every tile edge of the first 3 tiles, the last tile's first and last
    64 columns, and 256 random ones."""
    c = [np.arange(0, 41), np.arange(90, 141)]
    for t in (1, 2, 3):
        c.append(np.arange(t * rc.TILE - 3, t * rc.TILE + 4))
    last = (-(-P // rc.TILE) - 1) * rc.TILE
    c += [np.arange(last, last + 64), np.arange(P - 64, P), np.random.RandomState(seed).randint(0, P, 256)]
    c = np.unique(np.concatenate(c))
    return c[(c >= 0) & (c < P)]


_cache = {}


def _prepared(p):
    if p not in _cache:
        d = G.build(p)
        cols = sample_cols(p.P, p.seed)
        truth, mass = rc.truth_cols(d['table'], d['idx'], d['w'], cols)
        _cache.clear()
        _cache[p] = d, cols, truth, mass
    return _cache[p]


@pytest.mark.parametrize('p', G.PROBLEMS, ids=[p.id for p in G.PROBLEMS])
def test_emulated_kernel_order_passes(p):
    d, cols, truth, mass = _prepared(p)
    lay = rc.rc_layout(p.P, p.K, rc.H100_SMS)
    out = rc.emulate(d['table'], d['idx'], d['w'], p.P, lay, cols)
    worst, rms = rc.judge(out, truth, mass, lay)
    print(f'\n[rc f64 host] {p.id}: emulate worst/bound {worst:.3g} rms {rms:.3g}')
    assert rc.passes(worst, rms), (p.id, worst, rms)


def _groups():
    g = defaultdict(list)
    for p in G.PROBLEMS:
        g[p.group].append(p)
    return g


_GROUPS = _groups()


@pytest.mark.parametrize('group', list(_GROUPS))
def test_every_mutation_fails_some_problem_of_each_group(group):
    best = defaultdict(float)
    for p in _GROUPS[group]:
        d, cols, truth, mass = _prepared(p)
        lay = rc.rc_layout(p.P, p.K, rc.H100_SMS)
        for mu in rc.MUTATIONS:
            if rc.applicable(mu, p.P, p.K, lay):
                out = rc.emulate(d['table'], d['idx'], d['w'], p.P, lay, cols, mutation=mu)
                best[mu] = max(best[mu], rc.margin(*rc.judge(out, truth, mass, lay)))
    for mu, m in sorted(best.items(), key=lambda kv: kv[1]):
        print(f'\n[rc f64 host] {group}: {mu} {m:.3g}x')
    weakest = min(best, key=best.get)
    print(f'\n[rc f64 host] {group}: weakest mutation {weakest} {best[weakest]:.3g}x')
    missed = {mu: m for mu, m in best.items() if m < MUT_MIN}
    assert not missed, (group, missed)


def test_layout_restates_the_kernel_plan():
    """rc_layout at the edges the GPU cases are chosen for, and the kernel's two refusals."""
    assert rc.rc_layout(70659, 7200, 132) == rc.Layout(70, 1024, 8)                        # 1029 -> 1032, clamped to 1024
    assert rc.rc_layout(70659, 7168, 132) == rc.Layout(70, 1024, 7)                        # exactly 1024, unclamped
    assert rc.rc_layout(29393, 40000, 132) == rc.Layout(29, 1024, 40)
    assert rc.rc_layout(29393, 8, 132) == rc.Layout(29, 8, 1)
    assert rc.rc_layout(600_001, 10000, 132) == rc.Layout(586, 1024, 10)
    assert rc.rc_layout(4000 * 1024, 1024, 132) == rc.Layout(4000, 1024, 1)
    with pytest.raises(ValueError, match='ticket array'):
        rc.rc_layout(4000 * 1024, 1025, 132)
    with pytest.raises(ValueError, match='too many slice chunks'):
        rc.rc_layout(1, 1024 * 65536, 132)
    for p in G.PROBLEMS:
        lay = rc.rc_layout(p.P, p.K, rc.H100_SMS)
        sizes = rc.chunk_sizes(p.K, lay)
        assert sum(sizes) == p.K and min(sizes) >= 1 and max(sizes) <= lay.k_per_chunk <= rc.MAX_CHUNK
