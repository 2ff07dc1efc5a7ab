"""GPU: action noise on an env whose episodes end early, fused (es_rollout_closedloop_terminal_streams,
``BatchedRollout(fuse_noisy_terminal=True)``).

* the kernel against the per-evaluation route (es.py's _test_params_per_eval: numpy's gaussians drawn from a copy of the
  stream, one es_rollout_closedloop_terminal per evaluation, the stream advanced by what it consumed) at C = 1, 2 and 4 and
  flagrun's depth with E = 3, tanh and leaky ReLU, 0 and 1 coins, odd and even act, incoming streams with a cached gaussian,
  1, 3 and more streams than resident clusters, at fall heights from "half fall at step 0" to "nothing falls": indices, coin
  words, fitness, final positions, steps, noise_used, ObStat and the streams' key, position and has_gauss bit for bit, the
  cached gaussian to 1 ulp, and the noise trace against numpy's (randn * ac_std).astype(float32) at the positions consumed.
  An evaluation whose float32 noise differs from numpy's (CUDA's log) is reported, and its stream is compared up to it only;
* nothing falls: DeviceGeneration with fall_height=None (es_draw_noisy + the cluster kernel) bit for bit, cached gaussian
  included;
* es.step / es.test_params with the flag against the same calls without it (the per-evaluation route), two generations, with
  two rank streams and with the caller's one stream;
* MeanRewardResult falling at step 0 under the flag raises ZeroDivisionError with theta untouched;
* refusals: two coins per evaluation, a binned head at the ABI, a stream beyond the jump-ahead range."""
import ctypes as C
import math
import re
import warnings

import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib
from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu

SIGMA, AC_STD = 0.05, 0.01


def _activation(kind):
    from es_pytorch_b200.nn.nn import Activation
    return Activation(_lib.ES_ACT_LEAKY_RELU, float(np.float32(0.1))) if kind == 'leaky' else None


def _problem(eng, sizes, T, seed=7, gain=1.5):
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
    obs, act = sizes[0], sizes[-1]
    env = ClosedLoopEnv(obs, act, T)
    P = orc.n_params(orc.layer_dims(obs, list(sizes[1:-1]), act))
    rs = np.random.RandomState(seed)
    theta = np.concatenate([rs.randn(fi * fo + fo) * (gain / math.sqrt(fi)) for fi, fo in zip(sizes[:-1], sizes[1:])])
    table = rs.randn(P + 40_000).astype(np.float32)
    obs0, env_a, env_b = env.device_closed(eng)
    nr = np.random.RandomState(seed + 1)
    return dict(sizes=list(sizes), T=T, P=P, env=env, table=eng.to_device(table), theta=eng.to_device(theta.astype(np.float32)),
                mean=eng.to_device(nr.randn(obs) * 0.05), std=eng.to_device(0.5 + nr.rand(obs)), obs0=obs0, env_a=env_a,
                env_b=env_b, rew=eng.to_device(env.rew_vec[:T].copy()))


def _streams(seeds, pre):
    out = []
    for s, k in zip(seeds, pre):
        rs = np.random.RandomState(s)
        rs.randn(k)                                   # an odd count leaves a cached gaussian
        out.append(rs)
    return out


def _copy(streams):
    out = []
    for s in streams:
        c = np.random.RandomState()
        c.set_state(s.get_state())
        out.append(c)
    return out


def reference(eng, d, streams, n, coins, E, activation, h, chance=0.5):
    """The per-evaluation route, everything it computes kept per evaluation; advances ``streams`` as it does."""
    T, act, obs = d['T'], d['sizes'][-1], d['sizes'][0]
    f64, dev = torch.float64, eng.device
    fit, behv = torch.zeros(2, dtype=f64, device=dev), torch.zeros(2, 3, dtype=torch.float32, device=dev)
    steps, used = torch.zeros(2, 1, dtype=torch.int32, device=dev), torch.zeros(2, 1, dtype=torch.int64, device=dev)
    stats = torch.zeros(2 * obs + 2, dtype=f64, device=dev)
    idx0 = torch.zeros(1, dtype=torch.int64, device=dev)
    K = len(streams) * n
    r = dict(idx=np.zeros(K, np.int64), coins=np.zeros((K, 4), np.uint32), fit=np.zeros((2, K)), behv=np.zeros((2, K, 3), np.float32),
             steps=np.zeros((2, K), np.int64), used=np.zeros((2, K), np.int64), noise={}, osum=np.zeros(obs), osq=np.zeros(obs),
             ocount=0.0)
    upper = d['table'].numel() - d['P']
    for si, rs in enumerate(streams):
        for p in range(n):
            k = si * n + p
            r['idx'][k] = rs.randint(0, upper)
            w_pos, w_neg = eng.perturb(d['theta'], d['table'], torch.tensor([r['idx'][k]], dtype=torch.int64, device=dev), SIGMA)
            for sg, w in enumerate((w_pos, w_neg)):
                words = rs.randint(0, 2 ** 32, size=2 * coins, dtype=np.uint32) if coins else None
                if coins:
                    r['coins'][k, 2 * sg:2 * sg + 2] = words
                src = np.random.RandomState()
                src.set_state(rs.get_state())
                nz = (src.randn(E * T * act) * AC_STD).astype(np.float32)
                cw = None if words is None else eng.to_device(np.concatenate([words, words]).view(np.int32))
                stats.zero_()
                eng.rollout_closed_terminal(
                    d['table'], idx0, w.view(-1), 0.0, d['sizes'], d['mean'], d['std'], 1.0, d['obs0'], d['env_a'], d['env_b'],
                    d['rew'], d['env'].pos_scale, fit[0:1], fit[1:2], 1, behv[0], behv[1], coin_words=cw, save_obs_chance=chance,
                    ob_sum=stats[:obs] if coins else None, ob_sumsq=stats[obs:2 * obs] if coins else None,
                    ob_count=stats[2 * obs:] if coins else None, activation=activation,
                    act_noise=eng.to_device(np.stack([nz, nz]).reshape(1, 2, -1)), episodes=E, fall_height=h, steps=steps,
                    noise_used=used)
                hh = torch.cat([fit, behv[0].to(f64), steps[0].to(f64), used[0].to(f64), stats]).cpu().numpy()
                n_used = int(hh[6])
                rs.randn(n_used)
                r['fit'][sg, k], r['behv'][sg, k], r['steps'][sg, k], r['used'][sg, k] = hh[0], hh[2:5], int(hh[5]), n_used
                r['noise'][sg, k] = nz[:n_used]
                st = hh[7:] / 2
                if coins and st[2 * obs] > 0:                # ObStat.inc, evaluation by evaluation
                    r['osum'] += st[:obs]
                    r['osq'] += st[obs:2 * obs]
                    r['ocount'] += st[2 * obs]
    return r


def fused(eng, d, streams, n, coins, E, activation, h, chance=0.5, trace=True, T=None):
    """The new call on the streams' states; returns its outputs and the states it leaves."""
    T = T or d['T']
    act, obs, dev = d['sizes'][-1], d['sizes'][0], eng.device
    R = len(streams)
    st = [s.get_state() for s in streams]
    key = eng.to_device(np.stack([s[1] for s in st]).astype(np.uint32).view(np.int32))
    pos = eng.to_device(np.array([s[2] for s in st], np.int32))
    has = eng.to_device(np.array([s[3] for s in st], np.int32))
    gv = eng.to_device(np.array([s[4] for s in st], np.float64))
    K = R * n
    fit = torch.zeros(2, K, dtype=torch.float64, device=dev)
    behv = torch.zeros(2, K, 3, dtype=torch.float32, device=dev)
    stats = torch.zeros(2 * obs + 2, dtype=torch.float64, device=dev)
    used = torch.zeros(2, K, dtype=torch.int64, device=dev)
    tr = torch.full((K, 2, E * T * act), float('nan'), dtype=torch.float32, device=dev) if trace else None
    idx, cw, steps, _ = eng.rollout_closed_terminal_streams(
        key, pos, has, gv, n, d['table'].numel() - d['P'], coins, AC_STD, d['table'], d['theta'], SIGMA, d['sizes'], d['mean'],
        d['std'], 1.0, d['obs0'], d['env_a'], d['env_b'], d['rew'][:T].contiguous(), d['env'].pos_scale, fit[0], fit[1], 1,
        behv[0], behv[1], save_obs_chance=chance, ob_sum=stats[:obs] if coins else None,
        ob_sumsq=stats[obs:2 * obs] if coins else None, ob_count=stats[2 * obs:] if coins else None, episodes=E,
        activation=activation, fall_height=h, noise_used=used, noise_trace=tr)
    eng.sync()
    out = dict(idx=idx.cpu().numpy(), coins=None if cw is None else cw.cpu().numpy().view(np.uint32), fit=fit.cpu().numpy(),
               behv=behv.cpu().numpy(), steps=steps.cpu().numpy().astype(np.int64), used=used.cpu().numpy(),
               trace=None if tr is None else tr.cpu().numpy(), stats=stats.cpu().numpy())
    out['states'] = list(zip(key.cpu().numpy().view(np.uint32), pos.cpu().numpy(), has.cpu().numpy(), gv.cpu().numpy()))
    return out


def _h_low(eng, d, streams, n, coins, E, activation):
    """The median |z| after step 0 (the fused call with one step and nothing falling): about half the evaluations fall there."""
    o = fused(eng, d, _copy(streams), n, coins, 1, activation, 1e30, trace=False, T=1)
    return float(np.median(np.abs(o['behv'][..., 2])))


CASES = [
    # name, sizes, T, E, activation, coins, seeds, pre-drawn gaussians, pairs per stream
    ('c1_tanh', (15, 64, 64, 3), 60, 1, 'tanh', 1, [11, 12, 13], [0, 1, 3], 4),
    ('c1_leaky_even_act', (15, 64, 64, 4), 60, 2, 'leaky', 0, [21], [1], 5),
    ('simple_conf_c2', (15, 256, 256, 3), 50, 1, 'tanh', 1, [31, 32, 33], [1, 0, 0], 3),
    ('obj_c4_leaky', (17, 256, 256, 256, 6), 40, 1, 'leaky', 1, [41, 42], [0, 1], 2),
    ('flagrun_e3', (28, 128, 256, 256, 128, 8), 30, 3, 'tanh', 1, [51, 52, 53], [1, 0, 1], 2),
    ('many_streams', (15, 32, 32, 3), 20, 1, 'tanh', 1, list(range(600, 750)), [1, 0] * 75, 1),
]


@pytest.mark.parametrize('name,sizes,T,E,kind,coins,seeds,pre,n', CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize('height', ['low', 'mid', 'none'])
def test_kernel_is_the_per_evaluation_route(eng, name, sizes, T, E, kind, coins, seeds, pre, n, height):
    d = _problem(eng, sizes, T)
    act = _activation(kind)
    base = _streams(seeds, pre)
    lo = _h_low(eng, d, base, n, coins, E, act)
    h = {'low': lo, 'mid': lo * T / 4, 'none': 1e30}[height]
    h = float(np.float32(h))
    ref_streams = _copy(base)
    ref = reference(eng, d, ref_streams, n, coins, E, act, h)
    got = fused(eng, d, base, n, coins, E, act, h)
    K, R = len(seeds) * n, len(seeds)
    # the noise each evaluation added, against numpy's, in each stream's order: a differing value ends that stream's comparison
    upto = np.full(R, n)                                   # pairs of each stream compared bit for bit
    reported = []
    for s in range(R):
        for p in range(n):
            k = s * n + p
            bad = False
            for sg in range(2):
                u = ref['used'][sg, k]
                want, have = ref['noise'][sg, k], got['trace'][k, sg, :u]
                if got['used'][sg, k] == u and np.array_equal(want.view(np.uint32), have.view(np.uint32)):
                    continue
                diff = np.flatnonzero(want.view(np.uint32) != have[:len(want)].view(np.uint32)) if len(have) == len(want) else []
                if len(diff):
                    i = diff[0]
                    reported.append((s, p, sg, int(i), float(want[i]), float(have[i])))
                    bad = True
                    break
            if bad:
                upto[s] = p
                break
    if reported:
        warnings.warn(f'[{name}/{height}] float32 noise differing from numpy\'s (CUDA\'s log; stream, pair, sign, value index, '
                      f'numpy, device): {reported}; those streams are compared up to that evaluation')
        for (_, _, _, _, a, b) in reported:
            assert abs(np.float32(a) - np.float32(b)) <= np.spacing(np.float32(max(abs(a), abs(b))))
    keep = np.concatenate([np.arange(s * n, s * n + upto[s]) for s in range(R)]).astype(np.int64)
    assert np.array_equal(got['idx'][keep], ref['idx'][keep])
    if coins:
        assert np.array_equal(got['coins'][keep], ref['coins'][keep])
    for key in ('fit', 'steps', 'used'):
        assert np.array_equal(got[key][:, keep], ref[key][:, keep]), key
    assert np.array_equal(got['behv'][:, keep].view(np.uint32), ref['behv'][:, keep].view(np.uint32))
    fell0 = float(np.mean(got['steps'] == 0))
    ran = float(np.mean(got['steps'] + 1))
    print(f'\n[{name}/{height}] h {h:.4g}: fell at step 0 {fell0:.2f}, mean steps {ran:.1f} of {T}, pairs compared {len(keep)} of {K}')
    if height == 'none':
        assert np.all(got['steps'] == T - 1)
    if height == 'low':
        assert fell0 > 0
    if coins and not reported:                             # (a sum over every stream)
        obs = sizes[0]
        assert np.array_equal(got['stats'][:obs], ref['osum']) and np.array_equal(got['stats'][obs:2 * obs], ref['osq'])
        assert got['stats'][2 * obs] == ref['ocount']
    for s, (rs, st) in enumerate(zip(ref_streams, got['states'])):
        if upto[s] == n:                                   # the streams whose every noise value was numpy's
            want = rs.get_state()
            assert np.array_equal(st[0], want[1]) and st[1] == want[2] and st[2] == want[3], f'stream {s}'
            assert abs(st[3] - want[4]) <= np.spacing(abs(want[4])), f'stream {s}'


def _generation(eng, d, streams, h, E, act, coins=1):
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    env = d['env']
    obs_stream = eng.to_device(env.obs_stream[:d['T'] + 1].copy())
    return DeviceGeneration(d['table'], d['theta'].clone(), d['sizes'], obs_stream, d['rew'], streams, SIGMA, 0.005, Adam(d['P'], 0.01),
                            ob_clip=1.0, pos_scale=env.pos_scale, coins_per_eval=coins, save_obs_chance=0.5, engine=eng,
                            ac_std=AC_STD, closed=env.device_closed(eng), episodes=E, closed_act_noise=True, activation=act,
                            fall_height=h)


@pytest.mark.parametrize('sizes,E,kind', [((15, 256, 256, 3), 3, 'tanh'), ((15, 64, 64, 3), 1, 'leaky'),
                                          ((17, 256, 256, 256, 6), 2, 'tanh')], ids=['c2_tanh_e3', 'c1_leaky', 'c4_tanh_e2'])
def test_nothing_falls_is_the_drawn_ahead_generation_bit_for_bit(eng, sizes, E, kind):
    d = _problem(eng, sizes, 40)
    act = _activation(kind)
    seeds, pre = [71, 72, 73], [1, 0, 3]
    ga = _generation(eng, d, _streams(seeds, pre), None, E, act)
    gb = _generation(eng, d, _streams(seeds, pre), 1e30, E, act)
    for g in (ga, gb):
        g.set_obstat(d['mean'].cpu().numpy(), d['std'].cpu().numpy())
        g.evaluate(3)
    eng.sync()
    assert torch.equal(ga.idx, gb.idx) and torch.equal(ga.extras, gb.extras)
    assert torch.equal(ga.fit_local, gb.fit_local)
    assert torch.equal(ga._gen_stats[:2 * sizes[0] + 2], gb._gen_stats[:2 * sizes[0] + 2])
    assert torch.equal(ga.mt_state, gb.mt_state)                # key, position, has_gauss and the cached gaussian
    assert int(gb.steps_dev.min()) == 39


# ---------------------------------------------------------------------------------------------------- es.step / test_params
class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _setup(h, T=50, hidden=(32, 32), obs=15, act=3, seed=5, kind='tanh'):
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    env = ClosedLoopEnv(obs, act, T, fall_height=h)
    dims = orc.layer_dims(obs, hidden, act)
    P = orc.n_params(dims)
    rs = np.random.RandomState(seed)
    theta = np.concatenate([rs.randn(fi * fo + fo) * (1.5 / math.sqrt(fi)) for fi, fo in zip([obs, *hidden], [*hidden, act])])
    table = rs.randn(P + 40_000).astype(np.float32)

    def policy():
        net = FeedForward(list(hidden), torch.nn.LeakyReLU(0.1) if kind == 'leaky' else torch.nn.Tanh(), env, AC_STD, 5)
        p = Policy(net, 0.05, Adam(P, 0.01))
        p.flat_params[...] = theta.astype(np.float32)
        p.set_nn_params(p.flat_params)
        return p
    return env, policy, NoiseTable(P, table), P


@pytest.mark.parametrize('streams_kind', ['two_rank_streams', 'callers_stream'])
@pytest.mark.parametrize('kind', ['tanh', 'leaky'])
def test_es_step_with_the_flag_is_the_per_evaluation_route(eng, streams_kind, kind):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    T, n = 50, 3
    env, policy, nt, P = _setup(0.3, T, kind=kind)
    pa, pb = policy(), policy()
    two = streams_kind == 'two_rank_streams'
    sa, sb = _streams([31, 32], [1, 0]), _streams([31, 32], [1, 0])
    ra, rb = np.random.RandomState(41), np.random.RandomState(41)
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))      # n pairs per stream
    kw = dict(coins_per_eval=1, save_obs_chance=0.5, fuse_activations=kind == 'leaky')
    fa = BatchedRollout(env, T, rank_streams=sa if two else None, fuse_noisy_terminal=True, **kw)
    fb = BatchedRollout(env, T, rank_streams=sb if two else None, **kw)
    ka, kb = CenteredRanker(), CenteredRanker()
    assert es._can_fuse_step(dist.world(), pa, fa, ka) and not es._can_fuse_step(dist.world(), pb, fb, kb)

    class Steps(Reporter):
        def log_gen(self, fits, noiseless_tr, policy, steps, *args, **kw):
            self.steps = steps
    for g in range(2):
        rep_a, rep_b = Steps(), Steps()
        tra, oba = es.step(cfg, dist.world(), pa, nt, env, fa, ra, ka, rep_a)
        trb, obb = es.step(cfg, dist.world(), pb, nt, env, fb, rb, kb, rep_b)
        assert np.array_equal(np.asarray(ka.noise_inds), np.asarray(kb.noise_inds)), g
        assert np.array_equal(ka.fits_pos, kb.fits_pos) and np.array_equal(ka.fits_neg, kb.fits_neg), g
        assert np.array_equal(np.asarray(ka.ranked_fits), np.asarray(kb.ranked_fits)), g
        assert np.array_equal(pa.flat_params, pb.flat_params), g
        assert rep_a.steps == rep_b.steps, g
        assert oba.count == obb.count and np.array_equal(oba.sum, obb.sum) and np.array_equal(oba.sumsq, obb.sumsq), g
        assert tra.steps == trb.steps and np.array_equal(tra.result, trb.result), g
        assert np.array_equal(tra.positions, trb.positions), g
        for x, y in zip(sa + [ra], sb + [rb]):
            u, v = x.get_state(), y.get_state()
            assert np.array_equal(u[1], v[1]) and u[2:4] == v[2:4], g
            assert abs(u[4] - v[4]) <= np.spacing(abs(v[4])), g
        print(f'\n[fuse_noisy_terminal/{kind}/{streams_kind}] generation {g}: steps {rep_a.steps} of {2 * len(ka.noise_inds) * (T - 1)}')


def test_test_params_with_the_flag_is_the_per_evaluation_route(eng):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.obstat import ObStat
    T, n = 50, 4
    env, policy, nt, P = _setup(0.3, T)
    sa, sb = _streams([61, 62, 63], [0, 1, 1]), _streams([61, 62, 63], [0, 1, 1])
    oa, ob_ = ObStat(env.observation_space.shape, 0), ObStat(env.observation_space.shape, 0)
    fa = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.5, rank_streams=sa, fuse_noisy_terminal=True)
    fb = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.5, rank_streams=sb)
    pos, neg, inds, steps = es.test_params(dist.world(), n, policy(), nt, oa, fa, None)
    wpos, wneg, winds, wsteps = es.test_params(dist.world(), n, policy(), nt, ob_, fb, None)
    assert np.array_equal(inds, winds) and np.array_equal(pos, wpos) and np.array_equal(neg, wneg) and steps == wsteps
    assert oa.count == ob_.count and np.array_equal(oa.sum, ob_.sum) and np.array_equal(oa.sumsq, ob_.sumsq)
    for x, y in zip(sa, sb):
        u, v = x.get_state(), y.get_state()
        assert np.array_equal(u[1], v[1]) and u[2:4] == v[2:4]
        assert abs(u[4] - v[4]) <= np.spacing(abs(v[4]))


def test_mean_reward_falling_at_step_zero_raises_under_the_flag(eng):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.training_result import MeanRewardResult
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    T, n = 30, 4
    env, policy, nt, P = _setup(1e-30, T)
    p = policy()
    before = p.flat_params.copy()
    theta_dev = p.theta_dev(eng).clone()
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))
    fa = BatchedRollout(env, T, coins_per_eval=0, result=MeanRewardResult, fuse_noisy_terminal=True)
    ranker = CenteredRanker()
    assert not es._can_fuse_step(dist.world(), p, fa, ranker)
    with pytest.raises(ZeroDivisionError):
        es.step(cfg, dist.world(), p, nt, env, fa, np.random.RandomState(1), ranker, Reporter())
    assert np.array_equal(p.flat_params, before)
    assert torch.equal(p._theta_dev, theta_dev)


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_two_coins_per_evaluation_are_refused(eng):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.obstat import ObStat
    env, policy, nt, P = _setup(0.5, 30)
    fa = BatchedRollout(env, 30, coins_per_eval=2, save_obs_chance=0.5, fuse_noisy_terminal=True)
    with pytest.raises(ValueError, match='coins_per_eval'):
        es.test_params(dist.world(), 2, policy(), nt, ObStat(env.observation_space.shape, 0), fa, np.random.RandomState(1))
    d = _problem(eng, (15, 64, 64, 3), 30)
    with pytest.raises(ValueError, match='coins_per_eval'):
        fused(eng, d, _streams([1], [0]), 2, 2, 1, None, 0.5)


def _abi_call(eng, d, n_streams, n, bins=0, coins=0, E=1):
    """es_rollout_closedloop_terminal_streams straight through ctypes; returns (rc, message)."""
    lib, dev, T = eng.lib, eng.device, d['T']
    K = n_streams * n
    key = torch.zeros(n_streams, 624, dtype=torch.int32, device=dev)
    key[:, 0] = 1
    pos = torch.full((n_streams,), 624, dtype=torch.int32, device=dev)
    has = torch.zeros(n_streams, dtype=torch.int32, device=dev)
    gv = torch.zeros(n_streams, dtype=torch.float64, device=dev)
    idx = torch.zeros(K, dtype=torch.int64, device=dev)
    fit = torch.zeros(2, K, dtype=torch.float64, device=dev)
    steps = torch.zeros(2, K, dtype=torch.int32, device=dev)
    ls = (C.c_int * len(d['sizes']))(*d['sizes'])
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = lib.es_rollout_closedloop_terminal_streams(
        eng._ctx, p(key), p(pos), p(has), p(gv), n_streams, n, d['table'].numel() - d['P'], coins, AC_STD, p(d['table']),
        d['table'].numel(), p(d['theta']), d['P'], SIGMA, ls, len(d['sizes']) - 1, p(d['mean']), p(d['std']), 1.0, p(d['obs0']),
        p(d['env_a']), d['env_a'].shape[0], p(d['env_b']), p(d['rew']), T, d['env'].pos_scale, 0.5, p(idx), None, p(fit[0]), p(fit[1]),
        1, None, None, None, None, None, bins, _lib.ES_ACT_TANH, 0.0, E, 0.5, p(steps), None, None, eng.stream)
    return rc, lib.es_last_error().decode()


def test_abi_refuses_binned_heads_and_streams_beyond_the_jump_ahead_range(eng):
    d = _problem(eng, (15, 64, 64, 4), 1000)
    rc, msg = _abi_call(eng, d, 1, 1, bins=2)
    assert rc != 0 and 'binned' in msg
    # E T act = 10 x 1000 x 4 gaussians per evaluation: ~100 000 words, ~10 000 pairs exceed 2^20 blocks of one stream
    rc, msg = _abi_call(eng, d, 2, 10_000, E=10)
    assert rc != 0 and 'jump-ahead range' in msg, msg
    m = re.search(r'at most (\d+) pairs per stream fit, so the 20000 pairs need at least (\d+) streams', msg)
    assert m and 0 < int(m.group(1)) < 10_000 and int(m.group(2)) * int(m.group(1)) >= 20_000, msg
