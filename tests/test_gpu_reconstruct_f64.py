"""es_grad_reconstruct against a float64 truth (tests/rc_f64.py) at the shipped and benchmarked population sizes and at every
launch edge of reconstruct.cu: the shipped configs' parameter counts with K on both sides of the 1024-slice chunk clamp, column
counts at the lane / warp / tile edges, last chunks of 1 to 4 real slices, more column tiles than one wave holds, a table whose
byte offsets pass 2^31, and the tile tickets re-armed between launches of other layouts (and of a time-split rollout, which shares
them).

Every case asserts the layout it expects (rc_layout, from the kernel's plan) and one launch, so that a change of the plan fails here
instead of moving the case to another path.  The bounds are rc_f64.judge's: per column (k_per_chunk + n_chunks) U M_p, and the rms
over the columns below rc_f64.RMS_BOUND; tests/test_rc_f64_host.py shows on these same problems that every modelled kernel bug
exceeds one of them at least tenfold.
"""
from __future__ import annotations

import os
import sys
from typing import NamedTuple

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rc_f64 as rc  # noqa: E402

pytestmark = pytest.mark.gpu

SHIPPED_P = {'halfcheetah': 5702, 'humanoid': 29393, 'simple_conf': 70659, 'flagrun': 136456, 'obj': 137734}
SHIPPED_K = (1, 8, 4800, 10000, 40000)
EDGE_P = (1, 31, 32, 33, 127, 128, 129, 1023, 1024, 1025, 4097)
TABLE_EXTRA = 1_000_003
BIG_L = 2 ** 29 + 2 ** 20               # 2.1 GB of float32: byte offsets of the upper slices pass 2^31


class Problem(NamedTuple):
    group: str
    name: str
    P: int
    K: int
    seed: int

    @property
    def id(self):
        return f'{self.group}-{self.name}-P{self.P}-K{self.K}'


def _last_chunk_k(P, r, k_from):
    """The smallest K >= k_from whose last chunk has r real slices (at the H100's 132 SMs)."""
    K = k_from
    while True:
        lay = rc.rc_layout(P, K, rc.H100_SMS)
        if lay.n_chunks > 1 and rc.chunk_sizes(K, lay)[-1] == r:
            return K
        K += 1


def _problems():
    ps = []
    for name, P in SHIPPED_P.items():
        for K in SHIPPED_K:
            ps.append(Problem('shipped', name, P, K, P + K))
    for P in EDGE_P:
        ps.append(Problem('columns', 'edge', P, 3001, 7 * P + 1))
    for P in (5702, 29393):
        for r in (1, 2, 3, 4):
            ps.append(Problem('chunks', f'last{r}', P, _last_chunk_k(P, r, 3000), P + r))
    ps.append(Problem('chunks', 'kpc1024', 29393, 18 * 1024, 11))          # 18 chunks of exactly 1024, unclamped
    ps.append(Problem('chunks', 'kpc1024clamped', 29393, 18 * 1024 + 1, 12))   # 1028 clamped to 1024: 19 chunks, the last of 1
    ps.append(Problem('tiles', 'one_chunk_per_tile', 600_001, 10000, 13))   # 587 tiles: one chunk target, 10 chunks of 1024
    ps.append(Problem('tiles', 'single_chunk', 600_001, 5, 14))
    ps.append(Problem('tiles', 'max_tiles', 4000 * 1024, 1024, 15))         # 4000 tiles, one chunk: no tickets needed
    ps.append(Problem('large', 'offsets', 29393, 4800, 16))
    ps.append(Problem('large', 'offsets', 5702, 40000, 17))
    return ps


PROBLEMS = _problems()


def build(p: Problem):
    """numpy table (float32), idx (int64) and weights (float32, centered ranks of random fitnesses)."""
    from oracle import es_oracle as orc
    rs = np.random.RandomState(p.seed)
    P, K = p.P, p.K
    pos, neg = rs.randn(K), rs.randn(K)
    w = np.asarray(orc.centered_ranker(pos, neg)[0], dtype=np.float32).reshape(K)
    if p.group != 'large':
        L = P + TABLE_EXTRA
        table = rs.randn(L).astype(np.float32)
        idx = rs.randint(0, L - P, size=K).astype(np.int64)
        idx[0] = L - P - 1                                          # the last admissible slice
        if K > 2:
            idx[1] = idx[2]                                         # a duplicate
        return dict(table=table, idx=idx, w=w, L=L)
    # 2^29 + 2^20 floats; only two regions are filled: slices at the bottom and slices just above 2^29 floats (2^31 bytes)
    L = BIG_L
    table = np.zeros(L, dtype=np.float32)
    lo_end, hi_start = 1 << 22, (1 << 29) - (1 << 20)
    table[:lo_end + P] = rs.randn(lo_end + P).astype(np.float32)
    table[hi_start:] = rs.randn(L - hi_start).astype(np.float32)
    idx = np.where(rs.rand(K) < 0.5, rs.randint(0, lo_end, size=K), rs.randint(hi_start, L - P, size=K)).astype(np.int64)
    idx[:6] = [L - P - 1, 1 << 29, (1 << 29) + 1, (1 << 29) + 7, (1 << 29) - 1, 0]
    idx[6:10] = idx[1]                                              # duplicates
    w[::17] = 0.0                                                   # zero weights
    return dict(table=table, idx=idx, w=w, L=L)


def run_case(eng, dev_table, idx, w, P, expect):
    """One reconstruction: one launch, the expected layout; (out numpy, worst, rms) against the device float64 truth."""
    lay = rc.rc_layout(P, int(idx.numel()), eng.sm_count)
    assert lay == expect, (lay, expect)
    l0 = eng.launches
    out = eng.grad_reconstruct(dev_table, idx, w, P)
    eng.sync()
    assert eng.launches - l0 == 1
    truth, mass = rc.truth_device(dev_table, idx, w, P)
    worst, rms = rc.judge(out.cpu().numpy(), truth.cpu().numpy(), mass.cpu().numpy(), lay)
    torch.cuda.empty_cache()
    return out.cpu().numpy(), worst, rms


_seen = {}


@pytest.mark.parametrize('p', PROBLEMS, ids=[p.id for p in PROBLEMS])
def test_reconstruct_vs_float64(eng, p):
    d = build(p)
    expect = rc.rc_layout(p.P, p.K, rc.H100_SMS)                  # the plan the problem was chosen for
    t = eng.to_device(d['table'])
    out, worst, rms = run_case(eng, t, eng.to_device(d['idx']), eng.to_device(d['w']), p.P, expect)
    print(f'\n[rc f64] {p.id}: layout {tuple(expect)} worst/bound {worst:.3g} rms {rms:.3g}')
    _seen[p.id] = (worst, rms)
    assert np.all(np.isfinite(out))
    assert worst <= 1.0, (p.id, worst)
    assert rms <= rc.RMS_BOUND, (p.id, rms)


def test_too_many_tiles_is_refused(eng):
    from es_pytorch_b200._lib import EsLibraryError
    P, K = 4000 * 1024, 1025
    with pytest.raises(ValueError, match='ticket array'):
        rc.rc_layout(P, K, eng.sm_count)
    table = eng.zeros((P + 64,), torch.float32)
    idx = eng.zeros((K,), torch.int64)
    w = eng.zeros((K,), torch.float32)
    l0 = eng.launches
    with pytest.raises(EsLibraryError, match='P too large for the ticket array'):
        eng.grad_reconstruct(table, idx, w, P)
    assert eng.launches == l0


def test_tickets_rearm_across_layouts_and_a_time_split_rollout(eng):
    """Layouts A -> B -> A on one ctx, with a time-split F32 rollout (which takes its tickets from the same counters) between A and
    B: all three reconstructions meet the bounds, and the two A results are bit-identical."""
    from oracle import es_oracle as orc
    pa, pb = Problem('rearm', 'A', 29393, 10000, 21), Problem('rearm', 'B', 5702, 40000, 22)
    la, lb = rc.rc_layout(pa.P, pa.K, eng.sm_count), rc.rc_layout(pb.P, pb.K, eng.sm_count)
    assert la.n_chunks > 1 and lb.n_chunks > 1 and la.n_tiles != lb.n_tiles and la.n_chunks != lb.n_chunks
    da, db = build(pa), build(pb)
    ta, tb = eng.to_device(da['table']), eng.to_device(db['table'])
    args_a = (ta, eng.to_device(da['idx']), eng.to_device(da['w']), pa.P, la)
    out_a1, wa1, ra1 = run_case(eng, *args_a)
    # a time-split rollout: one policy pair, fewer policies than SMs
    rs = np.random.RandomState(3)
    obs_dim, act_dim, T = 17, 6, 1000
    dims = orc.layer_dims(obs_dim, (64, 64), act_dim)
    P = orc.n_params(dims)
    table = rs.randn(P + 5000).astype(np.float32)
    env = orc.SyntheticEnvSpec(obs_dim, act_dim, T)
    obsn = eng.normalise_obs(eng.to_device(env.obs_stream[:T]), eng.to_device(np.zeros(obs_dim)),
                             eng.to_device(np.ones(obs_dim)), 5.0)
    fit = torch.zeros(2, 1, dtype=torch.float64, device=eng.device)
    eng.rollout(eng.to_device(table), eng.to_device(np.array([7], dtype=np.int64)),
                eng.to_device((rs.randn(P) * 0.1).astype(np.float32)), 0.02, [obs_dim, 64, 64, act_dim], obsn,
                eng.to_device(env.rew_vec), env.pos_scale, fit[0], fit[1], 1)
    eng.sync()
    assert torch.isfinite(fit).all()
    _, wb, rb = run_case(eng, tb, eng.to_device(db['idx']), eng.to_device(db['w']), pb.P, lb)
    out_a2, wa2, ra2 = run_case(eng, *args_a)
    print(f'\n[rc f64] rearm: A {wa1:.3g}/{ra1:.3g}, B {wb:.3g}/{rb:.3g}')
    for worst, rms in ((wa1, ra1), (wb, rb), (wa2, ra2)):
        assert worst <= 1.0 and rms <= rc.RMS_BOUND
    assert np.array_equal(out_a1, out_a2)


def test_report_largest(eng):
    """The largest values of this module's cases against each bound (printed; the cases assert them)."""
    if _seen:
        w = max(_seen.items(), key=lambda kv: kv[1][0])
        r = max(_seen.items(), key=lambda kv: kv[1][1])
        print(f'\n[rc f64] largest worst/bound {w[1][0]:.3g} ({w[0]}), largest rms {r[1][1]:.3g} ({r[0]}) '
              f'over {len(_seen)} cases on {torch.cuda.get_device_name(0)}')
