"""GPU: episodes that end early on the closed-loop env (ClosedLoopEnv(fall_height=h), es_rollout_closedloop_terminal).

* the kernel against the float64 truth (tests/closed_f64.py with the fall height) at every shipped config's policy (C = 2 for 15-256-256-3,
  C = 4 for 17-256-256-256-6 and 28-128-256-256-128-8), a C = 1 shape, a binned head and a leaky-ReLU policy, at fall heights
  from "half fall at step 0" to "nothing falls".  Per evaluation: t_d exactly wherever the truth's |z| stays at least delta
  from h over the executed steps, delta the closed loop's position bound (2 ulp of the summed magnitude plus ACT_ERR
  pos_scale T: a kernel position within its bound decides each step as the truth does); the evaluations within delta (and,
  for the binned head, those whose top two outputs come within 1e-5) are counted, shown to be few, and skipped.  Fitness
  within the closed loop's EVAL_REL times the reward mass summed to t_d, the final position within its bound, steps, and
  the ObStat sums and count of the saved evaluations;
* nothing falls: bit for bit the fall_height=None result of the cluster kernel, also with action noise over E = 3 episodes
  (tanh and leaky ReLU at C = 1 and C = 2); at a shape fall_height=None runs on the one-CTA kernel, both within the float64
  bound;
* episodes: noise-free E = 3 is E = 1 bit for bit; with noise, E = 3 where an episode ends before an earlier one (the fold
  to the longest episode) against the truth, and the consumed gaussians sum_e (t_{d,e} + 1) act;
* es.test_params / es.step with ac_std = 0: the fused route against the same generation driven call by call with a python
  fit_fn through run_model's loop; with ac_std = 0.01, the per-evaluation route against the reference's loop, with two rank
  streams and with the caller's one stream over two generations (stream states exactly), and its refusal of two coins per
  evaluation;
* MeanRewardResult with an evaluation falling at step 0 raises ZeroDivisionError with theta untouched;
* dynamic scheduling: one launch equals the same evaluations launched a pair at a time."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib
from oracle import es_oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closed_f64 as cf  # noqa: E402
import f64_rollout as f64  # noqa: E402
from closed_f64 import ACT_ERR, EVAL_REL, OBS_ERR, U  # noqa: E402

pytestmark = pytest.mark.gpu

SIGMA = 0.02
LOW = np.array([-1.0, -0.5, -2.0], np.float32)
HIGH = np.array([1.0, 1.5, 0.5], np.float32)


def _head(kind):
    from es_pytorch_b200.nn.nn import Activation, BinnedHead
    if kind == 'binned':
        return BinnedHead(5, LOW.copy(), HIGH.copy()), None, (5, LOW, HIGH), np.tanh
    if kind == 'leaky':
        return None, Activation(_lib.ES_ACT_LEAKY_RELU, float(np.float32(0.1))), None, f64.leaky_relu(0.1)
    return None, None, None, np.tanh


def build(sizes, T, n_pairs=8, seed=3, g=1.0, band=8, E=1, ac_std=0.0, adim=None):
    P = orc.n_params(orc.layer_dims(sizes[0], sizes[1:-1], sizes[-1]))
    rs = np.random.RandomState(seed)
    table = rs.randn(P + 50_000).astype(np.float32)
    theta = np.concatenate([rs.randn(fi * fo + fo) * (g / math.sqrt(fi)) for fi, fo in zip(sizes[:-1], sizes[1:])]).astype(np.float32)
    idx = rs.randint(0, len(table) - P, size=n_pairs).astype(np.int64)
    act = adim or sizes[-1]
    spec = orc.ClosedLoopEnvSpec(sizes[0], act, T, band=band)
    nr = np.random.RandomState(seed + 1)
    noise = None
    if ac_std:
        noise = (np.random.RandomState(seed + 2).randn(n_pairs, 2, E * T * act) * ac_std).astype(np.float32)
    return dict(sizes=list(sizes), table=table, theta=theta, idx=idx, spec=spec, mean=nr.randn(sizes[0]) * 0.05,
                std=0.5 + nr.rand(sizes[0]), clip=1.0, noise=noise, E=E, obs0=spec.obs_stream[0].copy(),
                env_a=np.ascontiguousarray(spec.env_a.T), env_b=np.ascontiguousarray(spec.env_b.T), T=T, n=n_pairs)


def truth(d, h, binned=None, activation=np.tanh):
    s = d['spec']
    return cf.truth(d['table'], d['idx'], d['theta'], SIGMA, d['sizes'], d['mean'], d['std'], d['clip'], d['obs0'], d['env_a'],
                    d['env_b'], s.rew_vec, s.pos_scale, act_noise=d['noise'], episodes=d['E'], activation=activation,
                    fall_height=h, binned=binned)


def coins(n, saved):
    c = np.full((n, 4), 0xFFFFFFFF, dtype=np.uint32)
    for s, k in saved:
        c[k, 2 * s:2 * s + 2] = 0                                               # u = 0 < chance
    return c


def run(eng, d, h, head=None, activation=None, saved=(), pairs=None, terminal=True):
    """One call on the device (``pairs``: a sub-range of the problem's pairs): dict of fit, behv, steps, used, osum, osq,
    ocnt, launches."""
    n0, n1 = pairs or (0, d['n'])
    n, obs, dv = n1 - n0, d['sizes'][0], eng.to_device
    fit = torch.full((2, n), float('nan'), dtype=torch.float64, device=eng.device)
    behv = torch.full((2, n, 3), float('nan'), dtype=torch.float32, device=eng.device)
    steps = torch.full((2, n), -7, dtype=torch.int32, device=eng.device)
    used = torch.full((2, n), -7, dtype=torch.int64, device=eng.device)
    osum, osq = (torch.zeros(obs, dtype=torch.float64, device=eng.device) for _ in range(2))
    ocnt = torch.zeros(2, dtype=torch.float64, device=eng.device)
    s = d['spec']
    noise = None if d['noise'] is None else dv(np.ascontiguousarray(d['noise'][n0:n1]))
    cw = coins(d['n'], saved)[n0:n1]
    args = (dv(d['table']), dv(d['idx'][n0:n1]), dv(d['theta']), SIGMA, d['sizes'], dv(d['mean']), dv(d['std']), d['clip'],
            dv(d['obs0']), dv(d['env_a']), dv(d['env_b']), dv(s.rew_vec), s.pos_scale, fit[0], fit[1], 1, behv[0].view(-1),
            behv[1].view(-1))
    kw = dict(coin_words=dv(np.ascontiguousarray(cw).view(np.int32)), save_obs_chance=0.5, ob_sum=osum, ob_sumsq=osq,
              ob_count=ocnt, head=head, activation=activation, act_noise=noise, episodes=d['E'])
    l0 = eng.launches
    if terminal:
        eng.rollout_closed_terminal(*args, **kw, fall_height=h, steps=steps, noise_used=used if noise is not None else None)
    else:
        eng.rollout_closed_mlp(*args, **kw)
    eng.sync()
    return dict(fit=fit.cpu().numpy(), behv=behv.cpu().numpy(), steps=steps.cpu().numpy(), used=used.cpu().numpy(),
                osum=osum.cpu().numpy(), osq=osq.cpu().numpy(), ocnt=ocnt.cpu().numpy(), launches=eng.launches - l0)


def heights(d, binned=None, activation=np.tanh):
    """Fall heights from 'about half the evaluations fall at step 0' to 'nothing falls', from the never-falling truth."""
    tr = truth(d, 1e30, binned, activation)
    z0, zmax = tr['z0'].ravel(), tr['zmax'].ravel()
    return [float(np.median(z0)), float(np.quantile(zmax, 0.3)), float(np.quantile(zmax, 0.7)), float(2 * zmax.max() + 1e-3)]


def knife_edges(d, tr, T):
    """The evaluations whose fall the float32 kernel may decide differently from the truth: |z| within delta of h at some
    executed step (delta: the position bound), or, for a binned head, two top outputs within 1e-5."""
    ps = float(np.float32(d['spec'].pos_scale))
    delta = 2 * U * tr['mag'][..., 2] + ACT_ERR * ps * T
    return (tr['gap'] < delta) | (tr['margin'] < 1e-5), delta


def clear_of_knife_edges(d, h, binned=None, activation=np.tanh):
    """h, or a height up to a few percent above it where few evaluations sit on a knife edge (a binned head's positions take
    few distinct values, and a height picked among them lands on one), with its truth."""
    for _ in range(8):
        tr = truth(d, h, binned, activation)
        if knife_edges(d, tr, d['T'])[0].sum() <= 2:
            break
        h *= 1.0137
    return h, tr


def check(tag, d, h, got, tr, saved, T):
    """t_d where the truth is not within delta of a crossing (and not on a binned knife edge), then the values."""
    ps = float(np.float32(d['spec'].pos_scale))
    knife, delta = knife_edges(d, tr, T)
    ok = ~knife
    print(f'\n[closed terminal] {tag} h={h:.4g}: t_d {np.bincount(np.minimum(tr["steps"].ravel() * 4 // T, 4))} (quarters of T), '
          f'{int(knife.sum())} of {knife.size} within delta {delta.max():.2g} of a crossing')
    assert knife.sum() <= max(2, knife.size // 10), (tag, h, int(knife.sum()))
    assert np.array_equal(got['steps'][ok], tr['steps'][ok]), (tag, h)
    assert np.all(np.abs(got['fit'] - tr['fit'])[ok] <= (EVAL_REL * tr['mass'] + 1e-12)[ok]), (tag, h)
    bd = 2 * U * tr['mag'] + ACT_ERR * ps * T
    assert np.all((np.abs(got['behv'] - tr['behv']) <= bd)[ok]), (tag, h)
    m = np.zeros_like(ok)
    for s, k in saved:
        m[s, k] = True
    ns = max(1, len(saved))
    want_sum, want_sq = tr['osum'][m].sum(axis=0), tr['osq'][m].sum(axis=0)
    assert np.all(np.abs(got['osum'] - want_sum) <= 2 * T * U * tr['oabs'][m].sum(axis=0) + OBS_ERR * T * ns), (tag, h)
    assert np.all(np.abs(got['osq'] - want_sq) <= 2 * T * U * tr['osq'][m].sum(axis=0) + 2 * OBS_ERR * T * ns), (tag, h)
    assert got['ocnt'].tolist() == [float((tr['steps'][m] + 1).sum()), float(len(saved))], (tag, h)
    return ok


CASES = [  # name, sizes, T, head kind, cluster size
    ('simple_conf', (15, 256, 256, 3), 300, 'tanh', 2),
    ('obj', (17, 256, 256, 256, 6), 300, 'tanh', 4),
    ('flagrun', (28, 128, 256, 256, 128, 8), 300, 'tanh', 4),
    ('cta15', (15, 64, 64, 3), 300, 'tanh', 1),
    ('binned', (15, 64, 64, 15), 200, 'binned', 1),
    ('leaky', (17, 64, 64, 6), 200, 'leaky', 1),
]


@pytest.mark.parametrize('name,sizes,T,kind,C', CASES, ids=[c[0] for c in CASES])
def test_terminal_kernel_matches_the_float64_truth(eng, name, sizes, T, kind, C):
    head, activation, binned, f64_act = _head(kind)
    d = build(sizes, T, adim=3 if kind == 'binned' else None)
    assert eng.closed_mlp_plan(list(sizes), 8, head, activation)[0] in (C, 0)
    for h in heights(d, binned, f64_act):
        h, tr = clear_of_knife_edges(d, h, binned, f64_act)
        ok0 = ~knife_edges(d, tr, T)[0]
        saved = [(s, k) for s in range(2) for k in range(d['n']) if (k + s) % 2 == 0 and ok0[s, k]]
        got = run(eng, d, h, head, activation, saved)
        assert got['launches'] == 1
        check(name, d, h, got, tr, saved, T)


@pytest.mark.parametrize('name,sizes,kind', [('simple_conf', (15, 256, 256, 3), 'tanh'), ('obj', (17, 256, 256, 256, 6), 'tanh'),
                                             ('binned', (15, 64, 64, 15), 'binned'), ('leaky', (17, 64, 64, 6), 'leaky'),
                                             # action noise, E = 3: the noise offset and the episode fold
                                             ('noisy_c1', (15, 128, 64, 3), 'tanh+noise'),
                                             ('noisy_c2', (15, 256, 256, 3), 'tanh+noise'),
                                             ('noisy_leaky_c1', (17, 64, 64, 6), 'leaky+noise'),
                                             ('noisy_leaky_c2', (15, 256, 256, 3), 'leaky+noise')])
def test_nothing_falls_is_the_existing_kernels_bit_for_bit(eng, name, sizes, kind):
    kind, noisy = kind.split('+')[0], kind.endswith('+noise')
    head, activation, _, _ = _head(kind)
    T, E = 120, 3 if noisy else 1
    d = build(sizes, T, adim=3 if kind == 'binned' else None, E=E, ac_std=0.3 if noisy else 0.0)
    if noisy:
        assert eng.closed_mlp_plan(list(sizes), 8, head, activation)[0] == (2 if sizes[1] == 256 else 1)
    saved = [(s, k) for s in range(2) for k in range(d['n']) if (k + s) % 2 == 0]
    a = run(eng, d, 1e30, head, activation, saved)
    b = run(eng, d, None, head, activation, saved, terminal=False)
    for key in ('fit', 'behv', 'osum', 'osq', 'ocnt'):
        assert np.array_equal(a[key], b[key]), key
    assert (a['steps'] == T - 1).all()
    if noisy:
        assert (a['used'] == E * T * sizes[-1]).all()


def test_one_launch_equals_pairs_launched_one_at_a_time(eng):
    """Dynamic scheduling: which cluster runs which evaluation changes nothing."""
    d = build((15, 256, 256, 3), 200, n_pairs=40)
    h = heights(d)[1]
    whole = run(eng, d, h)
    for k in range(d['n']):
        one = run(eng, d, h, pairs=(k, k + 1))
        for key in ('fit', 'behv', 'steps'):
            assert np.array_equal(one[key][:, 0], whole[key][:, k]), (key, k)
    assert len(np.unique(whole['steps'])) > 3                # the evaluations end at many different steps


def test_episodes_without_noise_are_one_episode_bit_for_bit(eng):
    d1, d3 = build((17, 64, 64, 6), 150), build((17, 64, 64, 6), 150, E=3)
    h = heights(d1)[1]
    a, b = run(eng, d1, h), run(eng, d3, h)
    for key in ('fit', 'behv', 'steps'):
        assert np.array_equal(a[key], b[key]), key


@pytest.mark.parametrize('sizes', [(15, 64, 64, 3), (15, 256, 256, 3)])
def test_noisy_episodes_fold_to_the_longest_and_count_their_gaussians(eng, sizes):
    """E = 3 with action noise at a height where episodes of one evaluation end at different steps: some evaluation's
    last (or middle) episode ends before an earlier one, so the fold runs past the last episode's end."""
    E, T = 3, 150
    d = build(sizes, T, n_pairs=12, E=E, ac_std=0.3)
    tr0 = truth(d, 1e30)
    h = float(np.quantile(tr0['zmax'], 0.5))
    tr = truth(d, h)
    eps = tr['eps']
    shorter = (eps[..., 2] < eps[..., :2].max(axis=-1)) | (eps[..., 1] < eps[..., 0])
    saved = [(s, k) for s in range(2) for k in range(d['n']) if (k + s) % 2 == 0
             and tr['gap'][s, k] >= 2 * U * tr['mag'][s, k, 2] + ACT_ERR * 0.05 * T]
    got = run(eng, d, h, saved=saved)
    ok = check('noisy E=3', d, h, got, tr, saved, T)
    assert (shorter & ok).any(), eps
    act = sizes[-1]
    assert np.array_equal(got['used'][ok], ((eps + 1).sum(axis=-1) * act)[ok])


# ---------------------------------------------------------------------------------------------- es.test_params / es.step
class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _setup(h, T=60, hidden=(32, 32), ac_std=0.0, obs=15, act=3, seed=5):
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
        net = FeedForward(list(hidden), torch.nn.Tanh(), env, ac_std, 5)
        p = Policy(net, 0.05, Adam(P, 0.01))
        p.flat_params[...] = theta.astype(np.float32)
        p.set_nn_params(p.flat_params)
        return p
    return env, policy, NoiseTable(P, table), P


def _py_fit_fn(env, T, rs, chance, result_cls=None):
    """The scripts' fit_fn (simple_example.py:38, obj.py:53-63 with one episode): a coin, run_model's python loop."""
    from es_pytorch_b200.gym.gym_runner import run_model
    from es_pytorch_b200.gym.training_result import RewardResult
    cls = result_cls or RewardResult

    def fit(model, use_ac_noise=True):
        save = rs.random() < chance
        rews, behv, obs, steps = run_model(model, env, T, rs if use_ac_noise else None)
        return cls(rews, behv, obs if save else np.array([np.zeros(env.observation_space.shape)]), steps)
    return fit


def test_test_params_fused_against_the_python_loop(eng):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.obstat import ObStat
    T, n = 60, 6
    env, policy, nt, P = _setup(0.5, T)
    pa, pb = policy(), policy()
    ra, rb = np.random.RandomState(11), np.random.RandomState(11)
    oa, ob_ = ObStat(env.observation_space.shape, 0), ObStat(env.observation_space.shape, 0)
    fa = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.5)
    pos, neg, inds, steps = es.test_params(dist.world(), n, pa, nt, oa, fa, ra)
    wpos, wneg, winds, wsteps = es.test_params(dist.world(), n, pb, nt, ob_, _py_fit_fn(env, T, rb, 0.5), rb)
    assert np.array_equal(inds, winds)
    err = max(np.abs(pos - wpos).max(), np.abs(neg - wneg).max())
    print(f'\n[closed terminal] test_params fused vs python loop: max fitness err {err:.3g}, steps {steps} / {wsteps}')
    assert err <= 1e-4
    assert steps == wsteps and 0 < steps < 2 * n * (T - 1)      # they fell, after the first step
    assert oa.count == ob_.count
    assert np.allclose(oa.sum, ob_.sum, rtol=1e-5, atol=1e-4)
    sa, sb = ra.get_state(), rb.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2]


def test_es_step_fused_against_call_by_call(eng):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    T, n = 60, 6
    env, policy, nt, P = _setup(0.5, T)
    pa, pb = policy(), policy()
    ra, rb = np.random.RandomState(12), np.random.RandomState(12)
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))
    fa = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.5)
    ka, kb = CenteredRanker(), CenteredRanker()
    assert es._can_fuse_step(dist.world(), pa, fa, ka)

    class Steps(Reporter):
        def log_gen(self, fits, noiseless_tr, policy, steps, *args, **kw):
            self.steps = steps
    rep_a, rep_b = Steps(), Steps()
    tra, oba = es.step(cfg, dist.world(), pa, nt, env, fa, ra, ka, rep_a)
    trb, obb = es.step(cfg, dist.world(), pb, nt, env, _py_fit_fn(env, T, rb, 0.5), rb, kb, rep_b)
    assert np.array_equal(np.asarray(ka.noise_inds), np.asarray(kb.noise_inds))
    assert max(np.abs(ka.fits_pos - kb.fits_pos).max(), np.abs(ka.fits_neg - kb.fits_neg).max()) <= 1e-4
    if np.array_equal(np.asarray(ka.ranked_fits), np.asarray(kb.ranked_fits)):
        assert np.abs(pa.flat_params - pb.flat_params).max() <= 1e-5
    assert rep_a.steps == rep_b.steps
    assert oba.count == obb.count
    assert tra.steps == trb.steps and abs(tra.result[0] - trb.result[0]) <= 1e-4
    assert np.allclose(tra.positions[-3:], trb.positions[-3:], atol=1e-5)


def test_es_step_with_action_noise_and_two_streams_leaves_the_reference_states(eng):
    """ac_std = 0.01: the per-evaluation route.  The reference: two ranks each running es.py:67-74 with the scripts' fit_fn."""
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    T, n = 50, 3
    env, policy, nt, P = _setup(0.5, T, ac_std=0.01)
    pa, pb = policy(), policy()
    seeds = [31, 32]
    sa, sb = [np.random.RandomState(s) for s in seeds], [np.random.RandomState(s) for s in seeds]
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))     # n pairs per stream
    fa = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.5, rank_streams=sa)
    ranker = CenteredRanker()
    assert not es._can_fuse_step(dist.world(), pa, fa, ranker)
    es.step(cfg, dist.world(), pa, nt, env, fa, sa[0], ranker, Reporter())
    want_pos, want_neg, want_inds = [], [], []
    for rs in sb:
        fit = _py_fit_fn(env, T, rs, 0.5)
        for _ in range(n):
            idx, noise = nt.sample(rs)
            want_inds.append(idx)
            want_pos.append(fit(pb.pheno(noise)).result[0])
            want_neg.append(fit(pb.pheno(-noise)).result[0])
    assert np.array_equal(np.asarray(ranker.noise_inds), want_inds)
    err = max(np.abs(ranker.fits_pos.ravel() - want_pos).max(), np.abs(ranker.fits_neg.ravel() - want_neg).max())
    print(f'\n[closed terminal] noisy per-evaluation route: max fitness err {err:.3g}')
    assert err <= 1e-4
    # the noiseless evaluation of es.py:48 draws every stream's coin too
    for rs in sb:
        rs.random()
    for a, b in zip(sa, sb):
        x, y = a.get_state(), b.get_state()
        assert np.array_equal(x[1], y[1]) and x[2:] == y[2:]


def test_mean_reward_falling_at_step_zero_raises_before_anything_changes(eng):
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
    fa = BatchedRollout(env, T, coins_per_eval=0, result=MeanRewardResult)
    ranker = CenteredRanker()
    assert not es._can_fuse_step(dist.world(), p, fa, ranker)
    with pytest.raises(ZeroDivisionError):
        es.step(cfg, dist.world(), p, nt, env, fa, np.random.RandomState(1), ranker, Reporter())
    assert np.array_equal(p.flat_params, before)
    assert torch.equal(p._theta_dev, theta_dev)


def test_es_step_with_action_noise_and_one_stream_leaves_the_reference_state(eng):
    """ac_std = 0.01 with the caller's one ``rs`` (no rank_streams) and one coin per evaluation: the per-evaluation route must
    also hand the stream to the noiseless call of es.py:48, whose fit_fn draws its coin from it.  The reference: es.step with
    the scripts' fit_fn (the python loop), two generations, the stream's whole state compared after each."""
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    T, n = 50, 3
    env, policy, nt, P = _setup(0.5, T, ac_std=0.01)
    pa, pb = policy(), policy()
    ra, rb = np.random.RandomState(41), np.random.RandomState(41)
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))
    fa, fb = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.5), _py_fit_fn(env, T, rb, 0.5)
    ka, kb = CenteredRanker(), CenteredRanker()
    assert not es._can_fuse_step(dist.world(), pa, fa, ka)
    for g in range(2):
        tra, _ = es.step(cfg, dist.world(), pa, nt, env, fa, ra, ka, Reporter())
        trb, _ = es.step(cfg, dist.world(), pb, nt, env, fb, rb, kb, Reporter())
        assert np.array_equal(np.asarray(ka.noise_inds), np.asarray(kb.noise_inds)), g
        assert max(np.abs(ka.fits_pos - kb.fits_pos).max(), np.abs(ka.fits_neg - kb.fits_neg).max()) <= 1e-4, g
        assert np.array_equal(np.asarray(ka.ranked_fits), np.asarray(kb.ranked_fits)), g
        assert np.abs(pa.flat_params - pb.flat_params).max() <= 1e-5, g
        assert tra.steps == trb.steps and abs(tra.result[0] - trb.result[0]) <= 1e-4, g
        x, y = ra.get_state(), rb.get_state()
        assert np.array_equal(x[1], y[1]) and x[2:] == y[2:], g


def test_per_evaluation_route_refuses_two_coins_per_evaluation(eng):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.obstat import ObStat
    env, policy, nt, P = _setup(0.5, 30, ac_std=0.01)
    fa = BatchedRollout(env, 30, coins_per_eval=2, save_obs_chance=0.5)
    with pytest.raises(ValueError, match='coins_per_eval'):
        es.test_params(dist.world(), 2, policy(), nt, ObStat(env.observation_space.shape, 0), fa, np.random.RandomState(1))


def test_one_cta_shape_that_never_falls_agrees_within_the_float64_bound(eng):
    """At shapes es_rollout_closedloop_mlp runs on the one-CTA kernel (rollout_closed.cu, two FMA accumulators in the env
    step), the terminal call runs the cluster code: a never-falling env agrees with fall_height=None within the float64
    bound, not bit for bit.  Both against the truth, every evaluation running T steps."""
    sizes, T = (15, 64, 64, 3), 200
    assert eng.closed_mlp_plan(list(sizes), 8)[0] == 0                 # fall_height=None: the one-CTA kernel
    d = build(sizes, T)
    h = heights(d)[-1]
    tr = truth(d, h)
    assert (tr['steps'] == T - 1).all()
    saved = [(s, k) for s in range(2) for k in range(d['n']) if (k + s) % 2 == 0]
    for got in (run(eng, d, h, saved=saved), run(eng, d, None, saved=saved, terminal=False)):
        assert np.all(np.abs(got['fit'] - tr['fit']) <= EVAL_REL * tr['mass'])
        assert got['ocnt'].tolist() == [float(len(saved) * T), float(len(saved))]
