"""GPU: the generations bench.py times, at their real sizes, judged stage by stage (tests/gen_stages.py) against exact and
float64 references: draws, obs statistics, normalisation, fitness, novelty, rank weights, gradient sum and the Adam step.

The generations are built as bench.run_ours builds them (its WORKLOADS and VIRTUAL_RANKS_PER_GPU are read from bench.py): a
250 M-entry table torch.randn with seed 123, theta0 = RandomState(7).randn(P) * 0.1, streams RandomState(1000 + r), one save_obs
coin per evaluation at chance 0.01, sigma 0.02, l2coeff 0.005, Adam(lr 0.01):
  config 3   376-64-64-17, T = 1000, 8 streams x 1 250 pairs, ES_ROLLOUT_TC3 and ES_ROLLOUT_F32, three generations in a row; the
             third normalises with the statistics of the first two (set_obstat, as es.step's caller does);
  config 4   the same policy, 8 streams x 5 000 pairs (K = 40 000), TC3, one generation;
  config 5   NSRA: a 64-entry archive, k = 10, w = 0.5, TC3, two generations;
  noise      config 3 with ac_std = 0.01, TC3, one generation (the 340 M gaussians are replayed with numpy on the host);
  e2e        es.step with the bench's BatchedRollout against a DeviceGeneration from the same state, bit for bit.
Each generation's launches are asserted as restated from the host code (``_launches``).  The captured config-3 generation is
re-judged with modelled bugs applied on the host, each of which must be rejected.

Rank shifts against the float64 truth: the bounds (RANK_BOUNDS) are about twice the largest values measured on an H100 SXM
(80 GB HBM3, 700 W power limit).
"""
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_stages as gs  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from bench import VIRTUAL_RANKS_PER_GPU, WORKLOADS  # noqa: E402

WL = WORKLOADS['humanoid']
SIZES = [WL['obs'], *WL['hidden'], WL['act']]
T = WL['T']
P = sum(i * o + o for i, o in zip(SIZES[:-1], SIZES[1:]))
SIGMA, L2, LR, CHANCE = 0.02, 0.005, 0.01, 0.01
# (largest rank shift, largest |dw|) against the float64 truth's ranks, per population
# (measured: K = 10 000 at most a shift of 2 and |dw| 1.0e-4 = 2 / 19 999; K = 40 000 a shift of 3, |dw| 3.8e-5 = 3 / 79 999)
RANK_BOUNDS = {10000: (4, 4.5 / 19999), 40000: (6, 6.5 / 79999)}
T0 = time.perf_counter()


@pytest.fixture(scope='module')
def bench_inputs(eng):
    from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
    g = torch.Generator(device=eng.device).manual_seed(123)
    table = torch.randn(WL['table'], generator=g, device=eng.device, dtype=torch.float32)
    theta0 = (np.random.RandomState(7).randn(P) * 0.1).astype(np.float32)
    env = SyntheticEnv(WL['obs'], WL['act'], T)
    obs_dev, rew_dev = env.device_arrays(eng)
    yield dict(table=table, theta0=theta0, env=env, obs=obs_dev, rew=rew_dev)
    del table
    torch.cuda.empty_cache()


def _gen(eng, inp, mode, nsra=False, ac_std=0.0):
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    archive = np.random.RandomState(17).randn(64, 2) if nsra else None
    return DeviceGeneration(inp['table'], eng.to_device(inp['theta0'].copy()), SIZES, inp['obs'], inp['rew'],
                            [np.random.RandomState(1000 + r) for r in range(VIRTUAL_RANKS_PER_GPU)], SIGMA, L2, Adam(P, LR),
                            coins_per_eval=1, save_obs_chance=CHANCE, rollout_mode=mode, engine=eng,
                            archive=None if archive is None else eng.to_device(archive, torch.float64), nov_k=10, moo_w=0.5,
                            ac_std=ac_std)


def _streams(gen):
    R = gen.n_streams
    key = gen.mt_key.cpu().numpy().view(np.uint32)
    pos, has, gauss = gen.mt_pos.cpu().numpy(), gen.mt_has.cpu().numpy(), gen.mt_gauss.cpu().numpy()
    return [(key[r].copy(), int(pos[r]), int(has[r]), float(gauss[r])) for r in range(R)]


def _launches(gen, first: bool, shadows: int = 0, mt_lists: int = 0) -> int:
    """One DeviceGeneration.run of an open-loop generation, restated from the host code: the draw (es_draw_indices: 1;
    es_draw_noisy on its jump-ahead path: order, fill, flags, scan, walk, emit + the jump lists once per engine), the
    normalisation (1), the rollout (ES_ROLLOUT_TC3: prep + ubase + kernel, + the float16 shadows of a table the engine has
    not seen; ES_ROLLOUT_F32 at these sizes, the packed-FMA kernel: prep + ubase + kernel), novelty (1, with an archive), the
    obs statistics (the column sums on the first generation only, coin count + accumulate), the rank (keys, histogram, scan,
    scatter, finalise), the reconstruction (1) and Adam (1)."""
    n = (6 + mt_lists) if gen.ac_std else 1
    n += 1 + 3 + shadows
    n += 1 if gen.archive is not None else 0
    n += (1 if first else 0) + 2
    return n + 5 + 1 + 1


def _run(eng, gen, nps):
    """One generation; returns its Capture and its launch count."""
    eng.sync()
    opt = gen.optim
    st0 = dict(theta0=gen.theta.cpu().numpy().copy(), m0=opt.m.copy(), v0=opt.v.copy(), t0=opt.t, streams0=_streams(gen),
               ob_mean=gen.ob_mean.cpu().numpy().copy(), ob_std=gen.ob_std.cpu().numpy().copy())
    used = {}
    apply = gen.apply_optimizer

    def record(gsum, n_ranked):                          # what update() hands the optimizer as n_fits_ranked
        used['n_ranked'] = n_ranked
        apply(gsum, n_ranked)
    gen.apply_optimizer = record
    l0 = eng.launches
    gen.run(nps)
    eng.sync()
    launches = eng.launches - l0
    del gen.apply_optimizer
    cap = gs.Capture(sizes=SIZES, T=T, sigma=gen.sigma, l2coeff=gen.l2coeff, ob_clip=gen.ob_clip, pos_scale=gen.pos_scale,
                     save_obs_chance=gen.save_obs_chance, ac_std=gen.ac_std, lr=opt.lr, table=gen.table,
                     obs_stream=gen.obs_stream.cpu().numpy(), rew_vec=gen.rew_vec.cpu().numpy(),
                     idx=gen.idx.cpu().numpy(), coin_words=gen.extras.cpu().numpy().view(np.uint32).copy(),
                     obsn=gen.obsn.cpu().numpy(), fit=gen.fit_local.cpu().numpy(), stats=gen._gen_stats.cpu().numpy(),
                     weights=gen.weights.cpu().numpy(), n_ranked=int(used['n_ranked']), gsum=gen.gsum.cpu().numpy(),
                     theta1=gen.theta.cpu().numpy(), m1=opt.m.copy(), v1=opt.v.copy(), t1=opt.t, streams1=_streams(gen),
                     behv=None if gen.behv is None else gen.behv.cpu().numpy(),
                     act_noise=gen.act_noise if gen.ac_std else None,
                     archive=None if gen.archive is None else gen.archive.cpu().numpy(), nov_k=gen.nov_k, moo_w=gen.moo_w, **st0)
    return cap, launches


def _judge(eng, tag, cap, mode, truth=None):
    t = time.perf_counter()
    shift, dw = RANK_BOUNDS[cap.K]
    checks = gs.judge(cap, mode, eng.sm_count, shift, dw, truth=truth)
    print(f'\n{gs.report(tag, checks)}\n  ranks vs truth: {cap.extra.get("ranks_vs_truth")}, fitness error: {cap.extra.get("fitness")}, '
          f'saves {cap.extra.get("n_saved")}, '
          f'judged in {time.perf_counter() - t:.1f} s (file at {time.perf_counter() - T0:.0f} s)')
    gs.assert_ok(checks)
    return checks


def _obstat(caps):
    from oracle import es_oracle as orc
    obs = SIZES[0]
    st = orc.ObStatOracle((obs,), 1e-2)                 # Policy.update_obstat's running statistics (ObStat(shape, 1e-2))
    for c in caps:
        st.inc(c.stats[:obs], c.stats[obs:2 * obs], c.stats[2 * obs])
    return st.mean, st.std


_CONFIG3 = {}


def _config3(eng, inp, mode_name):
    """Three generations of config 3 (the third normalising with the statistics of the first two), each judged; every failed
    check is returned, per generation, for the caller to assert (computed once per mode)."""
    if mode_name in _CONFIG3:
        return _CONFIG3[mode_name]
    from es_pytorch_b200 import _lib
    mode = {'tc3': _lib.ES_ROLLOUT_TC3, 'f32': _lib.ES_ROLLOUT_F32}[mode_name]
    gen = _gen(eng, inp, mode)
    nps = WL['pairs'] // VIRTUAL_RANKS_PER_GPU
    caps, bad = [], []
    for g in range(3):
        if g == 2:
            mean, std = _obstat(caps)
            gen.set_obstat(mean, std)
        cap, nl = _run(eng, gen, nps)
        if g == 0 and mode == _lib.ES_ROLLOUT_TC3:
            assert nl - _launches(gen, True) in (0, 2), nl             # + hi and lo float16 shadows when this table is new
        else:
            assert nl == _launches(gen, g == 0), (g, nl)
        shift, dw = RANK_BOUNDS[cap.K]
        checks = gs.judge(cap, mode, eng.sm_count, shift, dw)
        print(f'\n{gs.report(f"config 3 {mode_name} generation {g + 1} ({nl} launches)", checks)}\n  ranks vs truth: '
              f'{cap.extra["ranks_vs_truth"]}, fitness error: {cap.extra["fitness"]}, saves {cap.extra["n_saved"]} '
              f'(file at {time.perf_counter() - T0:.0f} s)')
        bad.append(gs.failed(checks))
        if g == 2:
            assert not np.array_equal(cap.ob_std, np.ones_like(cap.ob_std))
        caps.append(cap)
        if g == 0 and mode_name == 'tc3':
            _not_vacuous(eng, cap, mode)
    del gen, caps
    torch.cuda.empty_cache()
    _CONFIG3[mode_name] = bad
    return bad


def test_config3_three_generations_f32(eng, bench_inputs):
    gs.assert_ok([c for b in _config3(eng, bench_inputs, 'f32') for c in b])


# The ES_ROLLOUT_TC3 fitness error against float64 carries a part proportional to the fitness: fitted over each population,
# e = kappa f + c + r with kappa = -8.3e-7 .. -8.7e-7 in every generation and config (ES_ROLLOUT_F32: |kappa| <= 9.4e-9), the magnitude
# shrink the wgmma chains' float32 accumulation is suspected of (the tanh epilogue is not its source: tanhf in its place measured
# the same; each layer's weight update adds to it in proportion to the fitness it gains).
# As Adam raises the mean fitness (-1.4, 461, 908 against a spread of 16-17), that relative error of a few float32 ulps grows
# against the spread: rms/spread 1.8e-6, 7.2e-6, 1.4e-5 (bound 8e-6), while the residual r stays at 1.37e-6 .. 1.45e-6 of the
# spread (configs 4, 5 and the noise variant: 1.37e-6 .. 1.38e-6) and the error per evaluation below 1e-7 of the reward mass.  A positive rescaling and a common offset change no rank.
# The residual and kappa are checked in every generation (gen_stages.stage_fitness); the plain rms/spread of generation 3 is
# the one known excess, asserted alone by the strict expected failure below.
TC3_KNOWN = {(2, 'fitness', 'rms/spread')}


def test_config3_three_generations_tc3(eng, bench_inputs):
    """Every check of every generation except the one known excess (TC3_KNOWN)."""
    bad = _config3(eng, bench_inputs, 'tc3')
    gs.assert_ok([c for g, b in enumerate(bad) for c in b if (g, c.stage, c.name) not in TC3_KNOWN])


@pytest.mark.xfail(strict=True, raises=gs.StageFailure,
                   reason='ES_ROLLOUT_TC3: a relative fitness error of ~8e-7, grown with the mean fitness to rms/spread 1.4e-5 '
                          'in generation 3 (bound 8e-6)')
def test_config3_tc3_generation3_rms_over_spread(eng, bench_inputs):
    """Only the known check: fails (as expected) while generation 3's plain rms/spread exceeds RMS_BOUND."""
    bad = _config3(eng, bench_inputs, 'tc3')
    gs.assert_ok([c for g, b in enumerate(bad) for c in b if (g, c.stage, c.name) in TC3_KNOWN])


def _not_vacuous(eng, cap, mode):
    """The captured config-3 outputs with modelled bugs applied on the host: each must be rejected."""
    truth = gs.fitness_truth(cap)
    for name in ('sign_swap', 'weights_next', 'drop_save'):
        what, mutate = gs.MUTATIONS[name]
        shift, dw = RANK_BOUNDS[cap.K]
        stages, margin = gs.rejection(gs.judge(mutate(cap), mode, eng.sm_count, shift, dw, truth=truth))
        print(f'  modelled bug at config 3, {what}: rejected by {stages}, margin {margin:.3g}x')
        assert stages is not None and margin >= 10, (name, stages, margin)


def test_config4_forty_thousand_pairs(eng, bench_inputs):
    from es_pytorch_b200 import _lib
    gen = _gen(eng, bench_inputs, _lib.ES_ROLLOUT_TC3)
    cap, nl = _run(eng, gen, WL['strong_total'] // VIRTUAL_RANKS_PER_GPU)
    assert cap.K == 40000 and nl - _launches(gen, True) in (0, 2), nl
    _judge(eng, f'config 4 tc3 ({nl} launches)', cap, _lib.ES_ROLLOUT_TC3)
    del gen
    torch.cuda.empty_cache()


def test_config5_nsra_two_generations(eng, bench_inputs):
    from es_pytorch_b200 import _lib
    wl = WORKLOADS['humanoid-nsra']
    assert wl.get('nsra') and wl['pairs'] == WL['pairs']
    gen = _gen(eng, bench_inputs, _lib.ES_ROLLOUT_TC3, nsra=True)
    for g in range(2):
        cap, nl = _run(eng, gen, wl['pairs'] // VIRTUAL_RANKS_PER_GPU)
        if g == 0:
            assert nl - _launches(gen, True) in (0, 2), nl
        else:
            assert nl == _launches(gen, False), nl
        assert cap.fit.shape == (2, wl['pairs'], 2)
        _judge(eng, f'config 5 nsra generation {g + 1} ({nl} launches)', cap, _lib.ES_ROLLOUT_TC3)
    del gen
    torch.cuda.empty_cache()


def test_config3_action_noise(eng, bench_inputs):
    from es_pytorch_b200 import _lib
    gen = _gen(eng, bench_inputs, _lib.ES_ROLLOUT_TC3, ac_std=0.01)
    cap, nl = _run(eng, gen, WL['pairs'] // VIRTUAL_RANKS_PER_GPU)
    extra = nl - _launches(gen, True)
    assert extra in (0, 1, 2, 3), nl                  # + the jump lists (1, once per engine) + the shadows of a new table (2)
    t = time.perf_counter()
    _judge(eng, f'config 3 tc3 ac_std 0.01 ({nl} launches)', cap, _lib.ES_ROLLOUT_TC3)
    print(f'  action noise: {cap.extra["noise_1ulp"]} of {cap.K * 2 * T * SIZES[-1]} gaussians one float32 ulp away next to a '
          f'midpoint; the whole judgement (the host replay of every stream included) took {time.perf_counter() - t:.1f} s')
    cap.act_noise = None
    del gen
    torch.cuda.empty_cache()


def test_e2e_step_equals_the_device_generation(eng, bench_inputs):
    """bench.py's e2e route (es.step, BatchedRollout over the 8 streams, the env resident on the device) from the state a
    DeviceGeneration starts from: indices, fitness, weights and theta' bit for bit, and the callers' streams where numpy's
    are after the generation's draws plus the noiseless evaluation's coin."""
    from es_pytorch_b200 import _lib, dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    from oracle import es_oracle as orc
    inp = bench_inputs
    nps = WL['pairs'] // VIRTUAL_RANKS_PER_GPU
    gen = _gen(eng, inp, _lib.ES_ROLLOUT_TC3)
    gen.run(nps)
    env = inp['env']
    net = FeedForward(list(WL['hidden']), torch.nn.Tanh(), env, 0.0, 5)
    policy = Policy(net, SIGMA, Adam(P, LR))
    policy.flat_params[...] = inp['theta0']
    nt = NoiseTable(P, inp['table'])
    streams = [np.random.RandomState(1000 + r) for r in range(VIRTUAL_RANKS_PER_GPU)]
    fit_fn = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=CHANCE, rank_streams=streams,
                            rollout_mode=_lib.ES_ROLLOUT_TC3, archive=None, nov_k=10)
    fit_fn.stream_env_from_host = False

    class _Cfg(dict):
        __getattr__ = dict.__getitem__
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * nps, batch_size=500), policy=_Cfg(l2coeff=L2))
    ranker = CenteredRanker()
    es.step(cfg, dist.world(), policy, nt, env, fit_fn, streams[0], ranker, Reporter())
    eng.sync()
    g2 = fit_fn._gen
    assert g2 is not gen and g2.K == gen.K == WL['pairs']
    assert torch.equal(g2.idx, gen.idx)
    assert np.array_equal(np.asarray(ranker.noise_inds).astype(np.int64), gen.idx.cpu().numpy())
    assert torch.equal(g2.fit_local, gen.fit_local)
    assert torch.equal(g2.weights, gen.weights)
    assert np.array_equal(np.asarray(ranker.ranked_fits).reshape(-1), gen.weights.cpu().numpy())
    assert np.array_equal(policy.flat_params, gen.theta.cpu().numpy())
    table_len = inp['table'].numel()
    for r, rs in enumerate(streams):
        ref = np.random.RandomState(1000 + r)
        for _ in range(nps):
            orc.sample_idx(table_len, ref, P)
            ref.random(); ref.random()
        ref.random()                                  # the noiseless evaluation's coin (es.py:48)
        a, b = rs.get_state(), ref.get_state()
        assert np.array_equal(a[1], b[1]) and a[2:] == b[2:], f'stream {r} after es.step'
    print(f'\ne2e es.step == DeviceGeneration at K = {gen.K}: indices, fitness, weights, theta bit for bit; streams exact '
          f'(file at {time.perf_counter() - T0:.0f} s)')
    del gen, g2, fit_fn
    torch.cuda.empty_cache()
