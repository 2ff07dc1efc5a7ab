"""The wide tensor-core rollout (rollout_tcw.cu: ES_ROLLOUT_TC3 / ES_ROLLOUT_TC for 2 to 4 hidden layers of widths in
{64, 128, 192, 256}, obs <= 256, act <= 32) against the float64 reference, with the bounds and the assert helper of
test_gpu_rollout_f64.py, at the shipped configs' policies and at its launch, tile and dispatch edges.

Launch counts are restated from the host launcher (``_tcw_chunk``): three launches per chunk of <= 256 MiB of weight images
(builder, rollout, finish)."""
import os
import sys

import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import f64_rollout as f64  # noqa: E402
import test_gpu_rollout_f64 as base  # noqa: E402

pytestmark = pytest.mark.gpu

TC, TC3 = _lib.ES_ROLLOUT_TC, _lib.ES_ROLLOUT_TC3
_MODES = [pytest.param(TC3, id='tc3'), pytest.param(TC, id='tc')]


def _cdiv(a, b):
    return -(-a // b)


def _tcw_chunk(sizes, mode):
    """rollout_tcw.cu's tw_run: pairs per launch chunk (<= 256 MiB of images of both signs)."""
    np_ = 2 if mode == TC3 else 1
    o = sum(_cdiv(fi, 64) * _cdiv(fo, 64) * np_ * 8192 for fi, fo in zip(sizes[:-1], sizes[1:]))
    o += sum(_cdiv(fo, 64) * 64 * 4 for fo in sizes[1:])
    img = (o + 1023) & ~1023
    return max(1, (256 << 20) // (2 * img))


def _tcw_launches(sizes, mode, n):
    return 3 * _cdiv(n, _tcw_chunk(sizes, mode))


# ---------------------------------------------------------------------------------------------- the shipped shapes
_SHIPPED = [
    # (name, sizes, T, E, n_pairs, fit_stride)
    ('simple_conf', [15, 256, 256, 3], 1000, 1, 40, 2),
    ('obj', [17, 256, 256, 256, 6], 1000, 1, 24, 1),
    ('obj-26', [26, 256, 256, 256, 6], 500, 1, 24, 1),
    ('obj-28', [28, 256, 256, 256, 8], 500, 1, 24, 1),
    ('flagrun', [28, 128, 256, 256, 128, 8], 500, 10, 20, 1),
    ('ns', [28, 256, 256, 256, 8], 10000, 1, 3, 1),
]


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('name,sizes,T,E,n,fit_stride', _SHIPPED, ids=[s[0] for s in _SHIPPED])
def test_wide_shipped_shapes(eng, mode, name, sizes, T, E, n, fit_stride):
    """Action noise (ac_std 0.01 as in the shipped configs), behaviour outputs, the NSRA fit_stride = 2 layout."""
    case = base.Case(eng, sizes, T, n, seed=sum(sizes) + T, E=E, ac_std=0.01)
    base._run_and_check(name, case, mode, base._sample(n, k=8), launches=_tcw_launches(sizes, mode, n),
                        fit_stride=fit_stride)


@pytest.mark.parametrize('mode,T', [(TC3, 1), (TC, 4)] + [(m, T) for m in (TC3, TC) for T in (127, 128, 129)])
def test_wide_episode_lengths(eng, mode, T):
    """T = 1 in TC3; T = 4, the shortest episode ES_ROLLOUT_TC takes on this path (test_wide_tc_refuses_short_episodes)."""
    case = base.Case(eng, [15, 256, 256, 3], T, 6, seed=T)
    base._run_and_check(f'wide T={T}', case, mode, list(range(6)), launches=3)


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('which', ['1', 'sm-1', 'chunk-1', 'chunk', 'chunk+1'])
def test_wide_pair_counts_and_chunks(eng, mode, which):
    """One pair, one below the SM count, and around the first launch-chunk boundary: pairs p0 - 1, p0, p0 + 1 of every
    boundary against the truth, and all pairs bit-identical to a run with the pairs reversed (no result depends on the
    grid or the chunking)."""
    sizes = [15, 256, 256, 3]
    c = _tcw_chunk(sizes, mode)
    n = {'1': 1, 'sm-1': eng.sm_count - 1, 'chunk-1': c - 1, 'chunk': c, 'chunk+1': c + 1}[which]
    case = base.Case(eng, sizes, 64, n, seed=n)
    bounds = [q for p0 in range(c, n, c) for q in (p0 - 1, p0, p0 + 1)]
    pairs = base._sample(n, bounds, k=max(8, len(bounds) + 3))
    f, b = base._run_and_check(f'wide n={n}', case, mode, pairs, launches=_tcw_launches(sizes, mode, n))
    if n > 1:
        fr, br, _ = case.run(mode, reverse=True)
        assert np.array_equal(f, fr) and np.array_equal(b, br)


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('sizes', [[7, 192, 64, 128, 1], [9, 128, 128, 32], [1, 64, 128, 4], [256, 256, 64, 5],
                                   [20, 64, 64, 64, 64, 2]],
                         ids=['mixed', 'act32', 'obs1', 'obs256', 'four-hidden-64'])
def test_wide_layer_shapes(eng, mode, sizes):
    n = 10
    case = base.Case(eng, sizes, 200, n, seed=sum(sizes))
    base._run_and_check(f'wide {sizes}', case, mode, list(range(n)), launches=3)


@pytest.mark.parametrize('mode', _MODES)
def test_wide_sigma_zero_signs_identical(eng, mode):
    case = base.Case(eng, [17, 256, 256, 256, 6], 300, 5, seed=0)
    case.sigma = 0.0
    f, b, _ = case.run(mode)
    assert np.array_equal(f[0], f[1]) and np.array_equal(b[0], b[1])
    # every evaluation is the same policy: the spread is 0, so only the per-evaluation bound applies
    tf, _, mass, _ = case.truth(list(range(5)))
    assert np.all(np.abs(f - tf) <= base.EVAL_REL[mode] * mass)


@pytest.mark.parametrize('mode', _MODES)
def test_wide_out_of_table_index(eng, mode):
    from es_pytorch_b200._lib import EsLibraryError
    case = base.Case(eng, [15, 256, 256, 3], 50, 3, seed=1)
    case.idx[1] = case.L - case.P                        # idx + P == L: NoiseTable.get's assert fails
    with pytest.raises(EsLibraryError, match='outside the table'):
        case.run(mode)
    eng.sync()


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('sizes', [[257, 256, 256, 3], [15, 256, 256, 33], [15, 96, 96, 3], [15, 256, 3]],
                         ids=['obs257', 'act33', 'width96', 'one-hidden'])
def test_wide_refusals(eng, mode, sizes):
    from es_pytorch_b200._lib import EsLibraryError
    P = f64.n_params(sizes)
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=eng.device)
    fit = torch.zeros(2, 1, dtype=torch.float64, device=eng.device)
    with pytest.raises(EsLibraryError, match=r'wide tensor-core path covers obs\(<=256\) with 2 to 4 hidden layers'):
        eng.rollout(z(P + 10), torch.zeros(1, dtype=torch.int64, device=eng.device), z(P), 0.02, sizes, z(8, sizes[0]),
                    z(8, sizes[-1]), 0.05, fit[0], fit[1], mode=mode)


@pytest.mark.parametrize('T', [1, 3])
def test_wide_tc_refuses_short_episodes(eng, T):
    """Single float16 products exceed ES_ROLLOUT_TC's per-evaluation bound on episodes of 1 to 3 steps (measured on an H100,
    see rollout_tcw.cu): refused, with TC3 named as the mode to use."""
    from es_pytorch_b200._lib import EsLibraryError
    case = base.Case(eng, [15, 256, 256, 3], T, 2, seed=T)
    with pytest.raises(EsLibraryError, match=r'needs T >= 4.*use ES_ROLLOUT_TC3'):
        case.run(TC)


@pytest.mark.parametrize('mode', _MODES)
def test_obs_64_64_act_stays_on_tc2(eng, mode):
    """obs-64-64-act keeps rollout_tc2.cu: with obs % 8 != 0 (no float16 shadows) that is prep + ubase + kernel = 3 launches
    for any number of pairs, where the wide launcher would take 3 per chunk."""
    sizes = [17, 64, 64, 6]
    n = 2 * _tcw_chunk(sizes, mode) + 1
    case = base.Case(eng, sizes, 64, n, seed=5)
    base._run_and_check('tc2 dispatch', case, mode, base._sample(n, k=8), launches=3)


def test_step_generations_at_the_simple_conf_shape_tc3(eng):
    """es.step on the single-synchronisation route with BatchedRollout(rollout_mode=ES_ROLLOUT_TC3) at simple_conf.json's
    policy (15-256-256-3), ac_std = 0.01, one save_obs coin per evaluation and two streams, for two generations.  Against
    the oracle's es_step: noise indices, the ObStat increments of the coins and the callers' RandomState objects (key,
    position, has_gauss) exact, the cached gaussian to 2 ulp.  Fitness against the float64 truth of the generation's own
    inputs (indices, theta, normalised observations, action noise) within the TC3 bounds.  parity_report is printed."""
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.generation import parity_report
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    from oracle import es_oracle as orc
    from test_gpu_generation import _Cfg, _api_objects
    obs_dim, act_dim, hidden, T, n = 15, 3, (256, 256), 200, 6
    sizes = [obs_dim, *hidden, act_dim]
    spec = orc.SyntheticEnvSpec(obs_dim, act_dim, T)
    dims = orc.layer_dims(obs_dim, hidden, act_dim)
    P = orc.n_params(dims)
    rs0 = np.random.RandomState(15)
    table, theta = rs0.randn(P + 400_000).astype(np.float32), (rs0.randn(P) * 0.1).astype(np.float32)
    env, net, policy, nt = _api_objects(eng, table, theta.copy(), spec, hidden)
    net._action_std = 0.01
    seeds = (151, 152)
    streams = [np.random.RandomState(s) for s in seeds]
    ref_streams = [np.random.RandomState(s) for s in seeds]
    fit_fn = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.25, rank_streams=streams, rollout_mode=TC3)
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))
    ranker = CenteredRanker()
    assert es._can_fuse_step(dist.world(), policy, fit_fn, ranker)
    flat, opt = theta.copy(), orc.AdamOracle(P, 0.01)
    stat = orc.ObStatOracle((obs_dim,), 1e-2)
    obmean, obstd = np.zeros(obs_dim), np.ones(obs_dim)
    for g in range(2):
        theta_g = policy.flat_params.copy()
        tr, gen_obstat = es.step(cfg, dist.world(), policy, nt, env, fit_fn, streams[0], ranker, Reporter())
        gen = fit_fn._gen
        idx, obsn, rew = gen.idx.cpu().numpy(), gen.obsn.cpu().numpy(), gen.rew_vec.cpu().numpy()
        k = gen.k_local
        noise = gen.act_noise.cpu().numpy().reshape(k, 2, 1, T, act_dim)
        print('\n[parity] generation', g, parity_report(gen, TC3))
        policy.update_obstat(gen_obstat)
        ref = orc.es_step(table, flat, opt, 0.02, dims, spec, ref_streams, n, obmean, obstd, 5.0, T, 500, 0.005, coins_per_eval=1,
                          save_obs_chance=0.25, batched=False, ac_std=0.01)
        stat.inc(ref['obstat'].sum, ref['obstat'].sumsq, ref['obstat'].count)
        obmean, obstd = stat.mean, stat.std
        assert np.array_equal(np.asarray(ranker.noise_inds), ref['inds']) and np.array_equal(idx, ref['inds'])
        assert np.array_equal(gen_obstat.sum, ref['obstat'].sum) and gen_obstat.count == ref['obstat'].count
        for a, b in zip(streams, ref_streams):
            sa, sb = a.get_state(), b.get_state()
            assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2] and sa[3] == sb[3], f'stream state after generation {g}'
            assert abs(sa[4] - sb[4]) <= 2 * np.spacing(abs(sb[4]))
        # the fitness of this generation against the float64 truth of its inputs
        case = base.Case.__new__(base.Case)
        case.sizes, case.T, case.n, case.E, case.P, case.L = sizes, T, k, 1, P, len(table)
        case.table, case.theta, case.idx, case.sigma, case.ps = table, theta_g, idx, 0.02, env.pos_scale
        case.obsn, case.rew, case.noise = obsn, rew, noise
        pairs = list(range(k))
        f = np.stack([np.asarray(ranker.fits_pos).reshape(-1), np.asarray(ranker.fits_neg).reshape(-1)])
        base._check(f'step generation {g}', TC3, case, f, None, pairs, case.truth(pairs))
        flat = policy.flat_params.copy()                 # the oracle continues from the device's theta
