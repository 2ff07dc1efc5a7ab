"""GPU: whole generations at the reference's shipped configs (configs/*.json), judged stage by stage (tests/gen_stages.py)
against exact and float64 references: draws, obs statistics, normalisation, fitness, novelty, rank weights, gradient sum and
the Adam step.

These configs run other code than the benchmarked ones: the wide tensor-core rollout (rollout_tcw.cu), the float32 rollout
with its weights staged in global memory in chunks of <= 256 MiB (rollout_f32.cu), ten episodes per evaluation, action-noise
streams of up to 300 x 2 x 80 000 gaussians, the NSR blend at w = 0, 0.5 and 1 with a 5-entry archive for k = 10, and the
closed-loop cluster kernel (rollout_closedw.cu), whose ObStat sums are float64 atomics in no fixed order.

Setup as test_gpu_generation_bench_configs.py: a 250 M-entry table torch.randn with seed 123, streams RandomState(1000 + r)
for 8 streams, sigma 0.02, l2coeff 0.005, Adam(lr 0.01), one save_obs coin per evaluation at chance 0.01.  Open-loop theta0
= RandomState(7).randn(P) * 0.1; closed-loop theta0 of scale 1 / sqrt(fan_in) (test_gpu_closed_f64.py's init regime).

Every case: the launches restated from the host code (``_launches``), the generation judged, then rerun from the same start
state and compared bit for bit (the closed loop's ObStat sums within the reordering bound of their float64 atomics).  One
captured generation per family (open loop with episodes, NSR, closed loop) is re-judged with the modelled bugs of its kind.

Rank shifts against the float64 truth (``RANK_BOUNDS``): about twice the largest values measured on an H100 SXM (80 GB HBM3,
700 W power limit), where the whole file took 285 s (the closed-loop flagrun truth on the CPU: 130 s of it).
"""
import math
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import closed_f64 as cf  # noqa: E402
import gen_stages as gs  # noqa: E402
import test_gpu_rollout_f64 as rf  # noqa: E402
import test_gpu_rollout_wide as rw  # noqa: E402

pytestmark = pytest.mark.gpu

# The reference's configs (the shapes: synthetic_env.KNOWN_SHAPES of the env each names):
#   configs/simple_conf.json  HopperBulletEnv-v0 (15, 3), hidden [256, 256], policies_per_gen 4800, max_steps 1000, ac_std 0.01
#   configs/nsra.json         HopperBulletEnv-v0 (15, 3), hidden [256, 256], policies_per_gen 9600, max_steps 2000, ac_std 0.01
#   configs/obj.json          HalfCheetah (17, 6), hidden [256, 256, 256], policies_per_gen 640, max_steps 1000, ac_std 0.01
#   configs/ns.json           Ant (28, 8), hidden [256, 256, 256], policies_per_gen 4800, max_steps 10000, ac_std 0.05
#   configs/flagrun.json      Ant (28, 8), hidden [128, 256, 256, 128], policies_per_gen 1200, max_steps 500, eps_per_policy 10
SHIPPED = {
    'simple_conf': dict(sizes=[15, 256, 256, 3], K=2400, T=1000, E=1, ac_std=0.01),
    'nsra': dict(sizes=[15, 256, 256, 3], K=4800, T=2000, E=1, ac_std=0.01),
    'obj': dict(sizes=[17, 256, 256, 256, 6], K=320, T=1000, E=1, ac_std=0.01),
    'ns': dict(sizes=[28, 256, 256, 256, 8], K=2400, T=10_000, E=1, ac_std=0.05),
    'flagrun': dict(sizes=[28, 128, 256, 256, 128, 8], K=600, T=500, E=10, ac_std=0.01),
}
STREAMS, TABLE, SIGMA, L2, LR, CHANCE, NOV_K = 8, 250_000_000, 0.02, 0.005, 0.01, 0.01, 10
# (largest rank shift, largest |dw|) against the float64 truth's ranks, per mode and population.  Measured: TC3 and F32 a shift
# of 1 at every K (|dw| = 1 / (2K - 1): 2.1e-4 at 2400, 1.0e-4 at 4800, 8.3e-4 at 600; ns at w = 0 ranks by novelty alone,
# |dw| 0; obj at K = 320 no rank differs); ES_ROLLOUT_TC (single float16 products) at simple_conf a shift of 12, |dw| 3.1e-3 (3504 of 4800 ranks differ)
RANK_BOUNDS = {('tc3', 2400): (2, 2.5 / 4799), ('tc3', 4800): (2, 2.5 / 9599), ('tc3', 320): (2, 2.5 / 639),
               ('tc3', 600): (2, 2.5 / 1199), ('f32', 2400): (2, 2.5 / 4799), ('f32', 600): (2, 2.5 / 1199),
               ('tc', 2400): (24, 6.3e-3)}
T0 = time.perf_counter()


@pytest.fixture(scope='module')
def table(eng):
    g = torch.Generator(device=eng.device).manual_seed(123)
    t = torch.randn(TABLE, generator=g, device=eng.device, dtype=torch.float32)
    yield t
    del t
    torch.cuda.empty_cache()


def _mode(name):
    from es_pytorch_b200 import _lib
    return {'tc3': _lib.ES_ROLLOUT_TC3, 'f32': _lib.ES_ROLLOUT_F32, 'tc': _lib.ES_ROLLOUT_TC}[name]


def _theta0(sizes, closed):
    P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
    rs = np.random.RandomState(7)
    if closed:
        return np.concatenate([rs.randn(fi * fo + fo) / math.sqrt(fi) for fi, fo in zip(sizes[:-1], sizes[1:])]).astype(np.float32)
    return (rs.randn(P) * 0.1).astype(np.float32)


def _archive(n):
    return np.random.RandomState(17).randn(n, 2)


class Setup:
    """The env and the device generation of one case, and how to rebuild it from a captured start state."""

    def __init__(self, eng, table, cfg, mode_name, archive=None, moo_w=0.5, closed=False, activation=None, rank_bounds=None):
        from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
        self.eng, self.table, self.cfg, self.mode_name = eng, table, cfg, mode_name
        # the policy's activation (an nn.Activation; None: tanh) and the rank-shift bounds it is judged by
        self.activation, self.rank_bounds = activation, RANK_BOUNDS if rank_bounds is None else rank_bounds
        self.sizes, self.T, self.E, self.ac_std = cfg['sizes'], cfg['T'], cfg['E'], cfg['ac_std']
        self.P = sum(i * o + o for i, o in zip(self.sizes[:-1], self.sizes[1:]))
        self.archive, self.moo_w, self.closed = archive, moo_w, closed
        self.env = (ClosedLoopEnv if closed else SyntheticEnv)(self.sizes[0], self.sizes[-1], self.T)
        self.obs, self.rew = self.env.device_arrays(eng)
        self.gen = self.make(_theta0(self.sizes, closed), None, [np.random.RandomState(1000 + r) for r in range(STREAMS)])

    def make(self, theta, adam_state, streams, ob=None):
        from es_pytorch_b200.generation import DeviceGeneration
        from es_pytorch_b200.nn.optimizers import Adam
        eng = self.eng
        opt = Adam(self.P, LR)
        if adam_state is not None:
            m, v, t = adam_state
            opt.state('m').copy_(torch.from_numpy(m).to(eng.device))
            opt.state('v').copy_(torch.from_numpy(v).to(eng.device))
            opt.t = t
        gen = DeviceGeneration(self.table, eng.to_device(theta.copy()), self.sizes, self.obs, self.rew, streams, SIGMA, L2, opt,
                               coins_per_eval=1, save_obs_chance=CHANCE, rollout_mode=_mode(self.mode_name), engine=eng,
                               archive=None if self.archive is None else eng.to_device(self.archive, torch.float64),
                               nov_k=NOV_K, moo_w=self.moo_w, ac_std=self.ac_std, episodes=self.E,
                               closed=self.env.device_closed(eng) if self.closed else None, closed_act_noise=self.closed,
                               activation=self.activation)
        if ob is not None:
            gen.set_obstat(*ob)
        return gen


def _streams(gen):
    key = gen.mt_key.cpu().numpy().view(np.uint32)
    pos, has, gauss = gen.mt_pos.cpu().numpy(), gen.mt_has.cpu().numpy(), gen.mt_gauss.cpu().numpy()
    return [(key[r].copy(), int(pos[r]), int(has[r]), float(gauss[r])) for r in range(gen.n_streams)]


def _rs(state):
    rs = np.random.RandomState()
    key, pos, has, gauss = state
    rs.set_state(('MT19937', key, pos, has, gauss))
    return rs


def _draw_launches(n_pairs, normals):
    """mt_gauss.cu's mg_plan: es_draw_noisy's jump-ahead path (order, fill, flags, scan, walk, emit: 6 launches) when a
    stream may consume >= 2048 blocks of 624 words, otherwise the sequential kernel and its finish (2)."""
    p_acc, n_acc = math.pi / 4, (normals + 1) // 2
    att_mean, att_sd = n_acc / p_acc, math.sqrt(n_acc * (1 - p_acc)) / p_acc
    evals = 2.0 * n_pairs
    words = 624 + n_pairs * (8 + 4) + 4 * (evals * att_mean + 12 * math.sqrt(evals) * att_sd + 64) + 2 * 5888 + 16 * 624
    return 6 if int(words / 624) + 1 >= 2048 else 2


def _rollout_launches(s: Setup, n):
    from es_pytorch_b200 import _lib
    if s.closed:
        return 1
    mode = _mode(s.mode_name)
    if mode == _lib.ES_ROLLOUT_F32:
        if s.activation is not None:                     # the general kernel only, never the packed-FMA one
            gw, chunk = rf._f32_layout(s.sizes)
            return 2 * -(-n // chunk) if gw else 1
        return rf._f32_launches(s.sizes, n, s.eng.sm_count)
    return rw._tcw_launches(s.sizes, mode, n)


def _launches(s: Setup, gen, first: bool) -> int:
    """One DeviceGeneration.run, restated from the host code: the draw (``_draw_launches``; without action noise the
    indices and coins alone, 1), the normalisation (1, open loop), the rollout (``_rollout_launches``: the wide tensor-core
    launcher's builder + rollout + finish per chunk, the staged float32 kernel's two per chunk, the closed loop's one
    cluster launch, which also accumulates the obs statistics), novelty (1, with an archive), the open loop's obs statistics
    (the column sums on the first generation only, coin count + accumulate), the rank (keys, histogram, scan, scatter,
    finalise), the reconstruction (1) and Adam (1).  Not counted: the jump lists (1, once per engine)."""
    n = _draw_launches(gen.k_local // gen.n_streams, s.E * s.T * s.sizes[-1]) if s.ac_std else 1     # es_draw_indices
    n += _rollout_launches(s, gen.k_local)
    if not s.closed:
        n += 1 + (1 if first else 0) + 2
    n += 1 if gen.archive is not None else 0
    return n + 5 + 1 + 1


def _run(s: Setup, gen, nps):
    eng = s.eng
    eng.sync()
    opt = gen.optim
    st0 = dict(theta0=gen.theta.cpu().numpy().copy(), m0=opt.m.copy(), v0=opt.v.copy(), t0=opt.t, streams0=_streams(gen),
               ob_mean=gen.ob_mean.cpu().numpy().copy(), ob_std=gen.ob_std.cpu().numpy().copy())
    used = {}
    apply = gen.apply_optimizer

    def record(gsum, n_ranked):
        used['n_ranked'] = n_ranked
        apply(gsum, n_ranked)
    gen.apply_optimizer = record
    l0 = eng.launches
    gen.run(nps)
    eng.sync()
    launches = eng.launches - l0
    del gen.apply_optimizer
    closed = {}
    if s.closed:
        obs0, env_a, env_b = s.env.device_closed(eng)
        closed = dict(obs0=obs0.cpu().numpy(), env_a=env_a.cpu().numpy(), env_b=env_b.cpu().numpy(), band=s.env.band)
    cap = gs.Capture(sizes=s.sizes, T=s.T, sigma=gen.sigma, l2coeff=gen.l2coeff, ob_clip=gen.ob_clip, pos_scale=gen.pos_scale,
                     save_obs_chance=gen.save_obs_chance, ac_std=gen.ac_std, lr=opt.lr, table=gen.table,
                     obs_stream=gen.obs_stream.cpu().numpy(), rew_vec=gen.rew_vec.cpu().numpy(),
                     idx=gen.idx.cpu().numpy(), coin_words=gen.extras.cpu().numpy().view(np.uint32).copy(),
                     obsn=None if s.closed else gen.obsn.cpu().numpy(), fit=gen.fit_local.cpu().numpy(),
                     stats=gen._gen_stats.cpu().numpy(), weights=gen.weights.cpu().numpy(), n_ranked=int(used['n_ranked']),
                     gsum=gen.gsum.cpu().numpy(), theta1=gen.theta.cpu().numpy(), m1=opt.m.copy(), v1=opt.v.copy(), t1=opt.t,
                     streams1=_streams(gen), behv=None if gen.behv is None else gen.behv.cpu().numpy(),
                     act_noise=gen.act_noise if gen.ac_std else None,
                     archive=None if gen.archive is None else gen.archive.cpu().numpy(), nov_k=gen.nov_k, moo_w=gen.moo_w,
                     episodes=gen.episodes, activation=s.activation, **closed, **st0)
    return cap, launches


def _judge(s: Setup, tag, cap, nl, truth=None):
    t = time.perf_counter()
    shift, dw = s.rank_bounds.get((s.mode_name, cap.K), (None, None))
    checks = gs.judge(cap, _mode(s.mode_name), s.eng.sm_count, shift, dw, truth=truth)
    print(f'\n{gs.report(f"{tag} ({nl} launches)", checks)}\n  ranks vs truth: {cap.extra.get("ranks_vs_truth")}, '
          f'fitness error: {cap.extra.get("fitness")}, saves {cap.extra.get("n_saved")}, '
          f'judged in {time.perf_counter() - t:.1f} s (file at {time.perf_counter() - T0:.0f} s)')
    return checks


def _check_launches(s, gen, nl, first):
    want = _launches(s, gen, first)
    if first:
        # + the jump lists (once per engine); the tensor-core modes + the float16 shadows of a table the engine has not seen
        assert nl - want in ((0, 1) if s.closed or s.mode_name == 'f32' else (0, 1, 2, 3)), (nl, want)
    else:
        assert nl == want, (nl, want)


def _stat_reorder_bound(cap):
    """|a - b| of two float64 sums of the same N = n_saved T terms in different orders: (N - 1) 2^-53 sum |term| each, twice."""
    tr = cap.extra['closed_truth']
    saved = gs.replayed_saves(cap)
    s_idx, j_idx = gs._truth_columns(tr, saved)
    N = max(1, len(s_idx) * cap.T)
    return (2 * N * 2.0 ** -53 * tr['oabs'][s_idx, j_idx].sum(axis=0),
            2 * N * 2.0 ** -53 * tr['osq'][s_idx, j_idx].sum(axis=0))


def _rerun_identical(s: Setup, cap, nps):
    """The generation again from its start state: everything bit for bit (closed loop: the ObStat sums within the reordering
    bound of their atomics, count and n_saved exact)."""
    gen = s.make(cap.theta0, (cap.m0, cap.v0, cap.t0), [_rs(st) for st in cap.streams0], (cap.ob_mean, cap.ob_std))
    c2, _ = _run(s, gen, nps)
    for name in ('idx', 'coin_words', 'fit', 'weights', 'gsum', 'theta1', 'm1', 'v1', 'behv'):
        a, b = getattr(cap, name), getattr(c2, name)
        assert (a is None and b is None) or np.array_equal(a, b), f'rerun: {name} differs'
    assert cap.n_ranked == c2.n_ranked and cap.t1 == c2.t1
    for a, b in zip(cap.streams1, c2.streams1):
        assert np.array_equal(a[0], b[0]) and a[1:] == b[1:], 'rerun: stream state differs'
    if cap.ac_std:
        assert torch.equal(cap.act_noise, c2.act_noise), 'rerun: action noise differs'
    obs = cap.obs_dim
    if s.closed:
        bs, bq = _stat_reorder_bound(cap)
        ds, dq = np.abs(cap.stats[:obs] - c2.stats[:obs]), np.abs(cap.stats[obs:2 * obs] - c2.stats[obs:2 * obs])
        assert np.all(ds <= bs) and np.all(dq <= bq), ('rerun: closed-loop ObStat beyond the reorder bound', (ds / bs).max())
        assert np.array_equal(cap.stats[2 * obs:], c2.stats[2 * obs:])
        print(f'  rerun: bit-identical; closed-loop ObStat sums differ by {(ds / bs).max():.3g} / {(dq / bq).max():.3g} of '
              f'the reorder bound')
    else:
        assert np.array_equal(cap.stats, c2.stats), 'rerun: obs statistics differ'
        print('  rerun: bit-identical')
    c2.act_noise = None
    del gen, c2
    torch.cuda.empty_cache()


def _not_vacuous(s: Setup, cap, names, truth=None):
    """The captured generation with modelled bugs applied on the host: each must be rejected by >= 10x."""
    if truth is None and not cap.closed:
        truth = gs.fitness_truth(cap)
    if cap.closed:
        truth = cap.extra['closed_truth']
    shift, dw = s.rank_bounds.get((s.mode_name, cap.K), (None, None))
    for name in names:
        what, mutate = gs.MUTATIONS[name]
        stages, margin = gs.rejection(gs.judge(mutate(cap), _mode(s.mode_name), s.eng.sm_count, shift, dw, truth=truth))
        print(f'  modelled bug, {what}: rejected by {stages}, margin {margin:.3g}x')
        assert stages is not None and margin >= 10, (name, stages, margin)


def _obstat(caps, obs):
    from oracle import es_oracle as orc
    st = orc.ObStatOracle((obs,), 1e-2)
    for c in caps:
        st.inc(c.stats[:obs], c.stats[obs:2 * obs], c.stats[2 * obs])
    return st.mean, st.std


def _case(eng, table, name, mode_name, generations=1, archive=None, moo_ws=(0.5,), archives=None, closed=False,
          mutations=(), mutate_gen=-1, cfg=None, activation=None, rank_bounds=None):
    """Run ``generations`` generations of config ``name``, judge each, re-judge generation ``mutate_gen`` with the modelled
    bugs ``mutations``, rerun the last one; every failed check returned, per generation.  ``activation``, ``rank_bounds``:
    as Setup's."""
    cfg = dict(SHIPPED[name] if cfg is None else cfg)
    s = Setup(eng, table, cfg, mode_name, archive=archive, moo_w=moo_ws[0], closed=closed, activation=activation,
              rank_bounds=rank_bounds)
    gen, nps = s.gen, cfg['K'] // STREAMS
    caps, bad = [], []
    for g in range(generations):
        if g > 0:
            gen.set_obstat(*_obstat(caps, s.sizes[0]))
            if archives is not None:
                s.archive = archives[g]
                gen.archive = eng.to_device(archives[g], torch.float64)
            s.moo_w = gen.moo_w = moo_ws[min(g, len(moo_ws) - 1)]
        cap, nl = _run(s, gen, nps)
        _check_launches(s, gen, nl, g == 0)
        checks = _judge(s, f'{name} {mode_name} generation {g + 1}', cap, nl)
        bad.append(gs.failed(checks))
        if g > 0:
            assert not np.array_equal(cap.ob_std, np.ones_like(cap.ob_std))
        caps.append(cap)
        if mutations and g == mutate_gen % generations:   # before the next generation overwrites the action-noise buffer
            _not_vacuous(s, cap, mutations)
    _rerun_identical(s, caps[-1], nps)
    for c in caps:
        c.act_noise = None
    del gen, caps
    s.gen = None
    torch.cuda.empty_cache()
    return bad


def _assert_ok(bad):
    gs.assert_ok([c for b in bad for c in b])


_CACHE = {}


def _simple_conf_tc3(eng, table):
    if 'simple_conf' not in _CACHE:
        _CACHE['simple_conf'] = _case(eng, table, 'simple_conf', 'tc3', generations=2)
    return _CACHE['simple_conf']


# As test_gpu_generation_bench_configs.TC3_KNOWN: ES_ROLLOUT_TC3's fitness error carries a part proportional to the fitness
# (kappa -0.6e-6 .. -1.3e-6 on the wide kernel at every shipped shape).  Once Adam has raised the mean fitness (simple_conf: 13.9
# to 148; nsra: -21 to 208) against a spread of ~10, that relative error reaches rms/spread 1.58e-5 (simple_conf) and 1.78e-5
# (nsra) in generation 2 (bound 8e-6), while the residual after the fitted scale and offset stays at 2.4e-6 of the spread.  A
# positive rescaling and a common offset change no rank.  Each is asserted alone by a strict expected failure.
TC3_KNOWN = {(1, 'fitness', 'rms/spread')}


def _known(bad, keep_known):
    return [c for g, b in enumerate(bad) for c in b if ((g, c.stage, c.name) in TC3_KNOWN) == keep_known]


def test_simple_conf_tc3_two_generations(eng, table):
    """Every check of both generations except the one known excess (TC3_KNOWN)."""
    gs.assert_ok(_known(_simple_conf_tc3(eng, table), False))


@pytest.mark.xfail(strict=True, raises=gs.StageFailure,
                   reason='ES_ROLLOUT_TC3: a relative fitness error of ~1e-6, grown with the mean fitness to rms/spread 1.6e-5 '
                          'in simple_conf generation 2 (bound 8e-6)')
def test_simple_conf_tc3_generation2_rms_over_spread(eng, table):
    gs.assert_ok(_known(_simple_conf_tc3(eng, table), True))


def test_simple_conf_f32_staged_weights(eng, table):
    gw, chunk = rf._f32_layout(SHIPPED['simple_conf']['sizes'])
    assert gw and SHIPPED['simple_conf']['K'] > chunk                 # staged weights, several launches
    _assert_ok(_case(eng, table, 'simple_conf', 'f32'))


def test_simple_conf_tc(eng, table):
    _assert_ok(_case(eng, table, 'simple_conf', 'tc'))


_NSRA = []


def _nsra(eng, table):
    """w = 1 with a 5-entry archive (k = 10: novelty over min(k, A) = 5), then w = 0.5 with the archive grown to 6; the
    modelled bugs on generation 1 (w = 1, where swapping w and 1 - w ranks by novelty alone).  Computed once."""
    if not _NSRA:
        a5, a6 = _archive(5), _archive(6)
        _NSRA.append(_case(eng, table, 'nsra', 'tc3', generations=2, archive=a5, archives=[a5, a6], moo_ws=(1.0, 0.5),
                           mutations=('novelty_over_reward', 'novelty_off_by_one', 'archive_clipped_to_k', 'moo_w_swapped'),
                           mutate_gen=0))
    return _NSRA[0]


def test_nsra_tc3_two_generations(eng, table):
    """Every check of both generations except the one known excess (TC3_KNOWN)."""
    gs.assert_ok(_known(_nsra(eng, table), False))


@pytest.mark.xfail(strict=True, raises=gs.StageFailure,
                   reason='ES_ROLLOUT_TC3: a relative fitness error of ~1e-6, grown with the mean fitness to rms/spread 1.8e-5 '
                          'in nsra generation 2 (bound 8e-6)')
def test_nsra_tc3_generation2_rms_over_spread(eng, table):
    """Only the known check: fails (as expected) while generation 2's plain rms/spread exceeds RMS_BOUND."""
    gs.assert_ok(_known(_nsra(eng, table), True))


def test_obj_tc3(eng, table):
    _assert_ok(_case(eng, table, 'obj', 'tc3'))


def test_ns_tc3(eng, table):
    """T = 10 000, ac_std 0.05, w = 0 (novelty alone ranks) with a 5-entry archive; the noise buffer is 1.5 GB."""
    _assert_ok(_case(eng, table, 'ns', 'tc3', archive=_archive(5), moo_ws=(0.0,)))


@pytest.mark.parametrize('mode_name', ['tc3', 'f32'])
def test_flagrun_ten_episodes(eng, table, mode_name):
    muts = ('episode0_noise', 'episodes_not_divided', 'first_episode_behaviour', 'sign_swap') if mode_name == 'tc3' else ()
    _assert_ok(_case(eng, table, 'flagrun', mode_name, mutations=muts))


@pytest.mark.parametrize('name,cluster', [('simple_conf', 2), ('flagrun', 4)])
def test_closed_loop(eng, table, name, cluster):
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
    cfg = SHIPPED[name]
    band = ClosedLoopEnv(cfg['sizes'][0], cfg['sizes'][-1], 2).band
    assert cf.plan(cfg['sizes'], band) == cluster and eng.closed_mlp_plan(cfg['sizes'], band)[0] == cluster
    muts = ('closed_obstat_pre_step', 'closed_count_t_minus_1', 'closed_drop_saved') if name == 'simple_conf' else ()
    _assert_ok(_case(eng, table, name, 'tc3', closed=True, mutations=muts))


def _e2e(eng, table, name, archive=None, moo_w=None, module=None, activation=None):
    """es.step (BatchedRollout over the 8 streams, the env resident on the device) against a DeviceGeneration from the same
    state: indices, fitness, weights and theta' bit for bit, and the callers' streams.  ``module``: the policy's activation
    module in place of tanh, ``activation`` its nn.Activation (es.step through BatchedRollout(fuse_activations=True))."""
    from es_pytorch_b200 import _lib, dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker, MultiObjectiveRanker
    from es_pytorch_b200.utils.reporters import Reporter
    cfg = SHIPPED[name]
    s = Setup(eng, table, cfg, 'tc3', archive=archive, moo_w=0.5 if moo_w is None else moo_w, activation=activation)
    nps = cfg['K'] // STREAMS
    gen = s.gen
    gen.run(nps)
    net = FeedForward(list(s.sizes[1:-1]), torch.nn.Tanh() if module is None else module, s.env, cfg['ac_std'], 5)
    assert (net.activation() if module is not None else None) == activation
    policy = Policy(net, SIGMA, Adam(s.P, LR))
    policy.flat_params[...] = _theta0(s.sizes, False)
    nt = NoiseTable(s.P, table)
    streams = [np.random.RandomState(1000 + r) for r in range(STREAMS)]
    fit_fn = BatchedRollout(s.env, s.T, coins_per_eval=1, save_obs_chance=CHANCE, rank_streams=streams,
                            rollout_mode=_lib.ES_ROLLOUT_TC3, archive=archive, nov_k=NOV_K, episodes=cfg['E'],
                            fuse_activations=module is not None)
    fit_fn.stream_env_from_host = False

    class _Cfg(dict):
        __getattr__ = dict.__getitem__
    ranker = CenteredRanker() if archive is None else MultiObjectiveRanker(CenteredRanker(), moo_w)
    es.step(_Cfg(general=_Cfg(policies_per_gen=2 * nps, batch_size=500), policy=_Cfg(l2coeff=L2)), dist.world(), policy, nt,
            s.env, fit_fn, streams[0], ranker, Reporter())
    eng.sync()
    g2 = fit_fn._gen
    assert g2 is not gen and g2.K == gen.K == cfg['K'] and g2.episodes == cfg['E'] and g2.activation == activation
    assert torch.equal(g2.idx, gen.idx) and torch.equal(g2.fit_local, gen.fit_local) and torch.equal(g2.weights, gen.weights)
    assert np.array_equal(np.asarray(ranker.noise_inds).astype(np.int64), gen.idx.cpu().numpy())
    assert np.array_equal(np.asarray(ranker.ranked_fits).reshape(-1), gen.weights.cpu().numpy())
    assert np.array_equal(policy.flat_params, gen.theta.cpu().numpy())
    # the callers' streams: the generation's draws (the device generation's end state) plus the noiseless evaluation's coin
    for r, (rs, st) in enumerate(zip(streams, _streams(gen))):
        ref = _rs(st)
        ref.random()
        a, b = rs.get_state(), ref.get_state()
        assert np.array_equal(a[1], b[1]) and a[2:4] == b[2:4] and a[4] == b[4], f'stream {r} after es.step'
    print(f'\ne2e {name}: es.step == DeviceGeneration at K = {gen.K}, E = {cfg["E"]}: indices, fitness, weights, theta bit for '
          f'bit; streams exact (file at {time.perf_counter() - T0:.0f} s)')
    gen.act_noise = g2.act_noise = None
    del gen, g2, fit_fn
    torch.cuda.empty_cache()


def test_e2e_step_flagrun_ten_episodes(eng, table):
    _e2e(eng, table, 'flagrun')


def test_e2e_step_nsra_multi_objective(eng, table):
    _e2e(eng, table, 'nsra', archive=_archive(5), moo_w=0.5)


def test_file_wall_time():
    print(f'\nshipped-config generations: file wall time {time.perf_counter() - T0:.0f} s')
