"""GPU: policies with ReLU, leaky-ReLU, ELU and sigmoid activations (es_rollout_*_activation) against the float64 truth.

* open loop, ES_ROLLOUT_F32 (the general float32 kernel) and ES_ROLLOUT_TC3 (the wide tensor-core kernel's code) at the
  shipped shapes, judged as the tanh kernels are (test_gpu_rollout_f64's EVAL_REL / RMS_BOUND / ACT_ERR against
  act_f64, f64_rollout's truth with the float64 activation); action noise and episodes, T = 1 and partial tiles, sigma = 0, pair counts
  around the SM count and multi-launch float32 chunks;
* closed loop at clusters of 1, 2 and 4 CTAs against act_f64.closed_truth (closed_f64's, with the activation; test_gpu_closed_f64's
  bounds), ObStat sums included;
* refusals (ES_ROLLOUT_TC, unknown kinds, a non-finite parameter, obs beyond TC3's coverage) and the float16 guard of TC3;
* ES_ACT_TANH through the new entry points is the old entry points bit for bit;
* es.test_params / es.step with BatchedRollout(fuse_activations=True): the DeviceGeneration's results bit for bit, and the
  python loop's within the float bound, with indices and stream states exact;
* every rerun is bit-identical (closed-loop ObStat sums within their atomics' reordering).
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib
from es_pytorch_b200.nn.nn import Activation

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import act_f64  # noqa: E402
import f64_rollout as f64  # noqa: E402
from test_gpu_rollout_f64 import ACT_ERR, EVAL_REL, RMS_BOUND, U, Case, _sample  # noqa: E402
import test_gpu_closed_f64 as cf  # noqa: E402

pytestmark = pytest.mark.gpu

F32, TC, TC3 = _lib.ES_ROLLOUT_F32, _lib.ES_ROLLOUT_TC, _lib.ES_ROLLOUT_TC3
ACTS = {
    'relu': (Activation(_lib.ES_ACT_RELU, 0.0), act_f64.relu),
    'leaky': (Activation(_lib.ES_ACT_LEAKY_RELU, float(np.float32(0.1))), act_f64.leaky_relu(0.1)),
    'elu': (Activation(_lib.ES_ACT_ELU, float(np.float32(0.7))), act_f64.elu(0.7)),
    'sigmoid': (Activation(_lib.ES_ACT_SIGMOID, 0.0), act_f64.sigmoid),
}
TANH = Activation(_lib.ES_ACT_TANH, 0.0)
# rms error over the checked evaluations relative to their fitness spread, about twice the largest value measured on an H100
# 80GB HBM3 (700 W power limit) over this file: F32 3.74e-6 (sigmoid at 376-64-64-17: its fast exponential and division),
# TC3 1.08e-5 (relu at 15-256-256-3: the split operands drop the lo * lo products, ~2^-22 of each, and an unbounded activation
# passes that relative error on at full size where tanh saturates).  Per evaluation the tanh files' EVAL_REL holds as it is
# (largest measured err / mass: F32 9.7e-7, TC3 1.8e-6)
RMS = {F32: 8e-6, TC3: 2.5e-5}
SHAPES = {'humanoid': [376, 64, 64, 17], 'simple_conf': [15, 256, 256, 3], 'obj': [17, 256, 256, 256, 6],
          'flagrun': [28, 128, 256, 256, 128, 8]}


class ActCase(Case):
    """test_gpu_rollout_f64's Case for a policy with activation ``name``."""

    def __init__(self, eng, name, sizes, T, n, seed, **kw):
        super().__init__(eng, sizes, T, n, seed, **kw)
        self.act, self.f64act = ACTS[name] if name != 'tanh' else (TANH, np.tanh)

    def run(self, mode, act=None, sigma=None):
        eng, n = self.eng, self.n
        fit = torch.full((2, n), float('nan'), dtype=torch.float64, device=eng.device)
        bh = torch.full((2, n, 3), float('nan'), dtype=torch.float32, device=eng.device)
        nz = None if self.noise is None else eng.to_device(self.noise)
        eng.rollout(self.d_table, eng.to_device(self.idx), self.d_theta, self.sigma if sigma is None else sigma, self.sizes,
                    self.d_obsn, self.d_rew, self.ps, fit[0], fit[1], 1, bh[0], bh[1], mode, act_noise=nz, episodes=self.E,
                    activation=self.act if act is None else act)
        eng.sync()
        f, b = fit.cpu().numpy(), bh.cpu().numpy()
        assert not np.isnan(f).any() and not np.isnan(b).any(), 'an evaluation was not written'
        return f, b

    def truth(self, pairs):
        return act_f64.rollout_f64(self.table, self.idx, self.theta, self.sigma, self.sizes, self.obsn, self.rew, self.ps,
                                   self.f64act, self.noise, self.E, pairs)


def _check(tag, mode, case, f, b, pairs, rms_check=True):
    tf, tb, mass, mag = case.truth(pairs)
    f, b = f[:, pairs], b[:, pairs]
    err = np.abs(f - tf)
    spread = max(tf.std(), 1e-3 * math.sqrt(case.T))
    rms = math.sqrt((err ** 2).mean())
    worst = (err / mass).max()
    print(f'\n[act f64] {tag} mode={mode}: rms/spread {rms / spread:.3g} (bound {RMS[mode]:.3g}), max err/mass {worst:.3g} '
          f'(bound {EVAL_REL[mode]:.3g})')
    assert np.all(err <= EVAL_REL[mode] * mass), (tag, worst)
    assert not rms_check or rms <= RMS[mode] * spread, (tag, rms / spread)
    tol = 2 * U * mag + ACT_ERR[mode] * case.ps * case.T
    assert np.all(np.abs(b - tb) <= tol), (tag, np.abs(b - tb).max())


def _run_check(tag, case, mode, pairs=None, repeat=True):
    f, b = case.run(mode)
    _check(tag, mode, case, f, b, list(range(case.n)) if pairs is None else pairs)
    if repeat:
        f2, b2 = case.run(mode)
        assert np.array_equal(f, f2) and np.array_equal(b, b2), f'{tag}: a rerun differs'
    return f, b


# ------------------------------------------------------------------------------------------------ open loop against float64
@pytest.mark.parametrize('mode', [F32, TC3], ids=['F32', 'TC3'])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('name', list(ACTS))
def test_open_loop_against_float64(eng, name, shape, mode):
    sizes = SHAPES[shape]
    case = ActCase(eng, name, sizes, 300, 12, seed=10 * list(ACTS).index(name) + list(SHAPES).index(shape))
    if mode == TC3 and sizes[0] > 256:
        # the wide kernel's activation buffer holds 256 input columns: obs 376 is refused, ES_ROLLOUT_F32 takes it
        with pytest.raises(_lib.EsLibraryError, match=r'obs 376.*ES_ROLLOUT_F32'):
            case.run(mode)
        return
    _run_check(f'{name} {shape}', case, mode)


@pytest.mark.parametrize('mode', [F32, TC3], ids=['F32', 'TC3'])
@pytest.mark.parametrize('name', ['relu', 'elu', 'sigmoid'])
def test_action_noise_and_episodes(eng, name, mode):
    case = ActCase(eng, name, [15, 256, 256, 3], 200, 10, seed=5, E=3, ac_std=0.1)
    _run_check(f'{name} E=3 noisy', case, mode)
    case = ActCase(eng, name, [28, 128, 256, 256, 128, 8], 150, 6, seed=6, E=1, ac_std=0.05)
    _run_check(f'{name} E=1 noisy', case, mode)


@pytest.mark.parametrize('mode', [F32, TC3], ids=['F32', 'TC3'])
@pytest.mark.parametrize('T', [1, 2, 127, 129, 257])
def test_episode_lengths_and_partial_tiles(eng, T, mode):
    _run_check(f'leaky T={T}', ActCase(eng, 'leaky', [17, 64, 64, 6], T, 8, seed=T), mode)


@pytest.mark.parametrize('mode', [F32, TC3], ids=['F32', 'TC3'])
def test_sigma_zero_gives_identical_signs(eng, mode):
    for name in ACTS:
        case = ActCase(eng, name, [15, 256, 256, 3], 100, 4, seed=9)
        f, b = case.run(mode, sigma=0.0)
        assert np.array_equal(f[0], f[1]) and np.array_equal(b[0], b[1]), name


def test_pair_counts_around_the_sm_count_and_float32_chunks(eng):
    sm = eng.sm_count
    for n in (sm // 2 - 1, sm // 2, sm // 2 + 1, sm + 1):
        case = ActCase(eng, 'relu', [17, 64, 64, 6], 64, n, seed=n)
        for mode in (F32, TC3):
            _run_check(f'relu n={n}', case, mode, pairs=_sample(n, k=12), repeat=False)
    # 15-256-256-3's staged weights (2 x 285 KiB per pair): 256 MiB chunks of 459 pairs, so 487 pairs take two launches
    case = ActCase(eng, 'elu', [15, 256, 256, 3], 40, 487, seed=3)
    l0 = eng.launches
    _run_check('elu two F32 chunks', case, F32, pairs=_sample(487, must=(485, 486), k=10), repeat=False)
    assert eng.launches - l0 == 4                        # two chunks, each a staging and a rollout launch


# ------------------------------------------------------------------------------------------------ refusals and the float16 guard
def test_refusals(eng):
    case = ActCase(eng, 'relu', [15, 256, 256, 3], 16, 2, seed=1)
    with pytest.raises(_lib.EsLibraryError, match=r'code -3.*ES_ROLLOUT_TC refuses'):
        case.run(TC)
    for bad in (Activation(7, 0.0), Activation(-1, 0.0)):
        with pytest.raises(_lib.EsLibraryError, match=r'code -1.*unknown activation'):
            case.run(F32, act=bad)
    with pytest.raises(_lib.EsLibraryError, match=r'code -1.*must be finite'):
        case.run(F32, act=Activation(_lib.ES_ACT_LEAKY_RELU, float('nan')))
    with pytest.raises(_lib.EsLibraryError, match=r'hidden layer 1 of width 100'):
        ActCase(eng, 'relu', [15, 100, 64, 3], 16, 2, seed=1).run(TC3)
    # the engine is usable afterwards
    _run_check('after refusals', case, F32, repeat=False)


def test_tc3_flags_hidden_values_beyond_float16_and_f32_takes_them(eng):
    case = ActCase(eng, 'relu', [15, 256, 256, 3], 50, 4, seed=2)
    case.theta = (case.theta.astype(np.float64) * 1000).astype(np.float32)
    case.d_theta = eng.to_device(case.theta)
    # the premise: the second hidden layer of theta itself leaves float16 range
    h = case.obsn.astype(np.float64)
    for wo, bo, fi, fo in f64.layer_slices(case.sizes)[:2]:
        h = np.maximum(h @ case.theta[wo:wo + fi * fo].reshape(fo, fi).T.astype(np.float64) + case.theta[bo:bo + fo], 0.0)
    assert np.abs(h).max() > 4 * 65504
    f, b = case.run(F32)
    # (per evaluation only: hidden values beyond 1e5 leave a fitness spread small against the reward mass)
    _check('relu x1000 F32', F32, case, f, b, list(range(case.n)), rms_check=False)
    with pytest.raises(_lib.EsLibraryError, match=r'float16 range'):
        case.run(TC3)
    assert eng.lib.es_check_async(eng._ctx) == 0          # reported once
    f2, b2 = case.run(F32)
    assert np.array_equal(f, f2)


# ------------------------------------------------------------------------------------------------ tanh through the new entry points
@pytest.mark.parametrize('mode', [F32, TC, TC3], ids=['F32', 'TC', 'TC3'])
@pytest.mark.parametrize('shape', ['humanoid', 'simple_conf'])
def test_tanh_through_the_new_entry_point_is_the_old_one(eng, shape, mode):
    case = ActCase(eng, 'tanh', SHAPES[shape], 130, 9, seed=4, E=2, ac_std=0.05)
    fa, ba = case.run(mode, act=TANH)
    fb, bb = _old(case, mode)
    assert np.array_equal(fa, fb) and np.array_equal(ba, bb)


def _old(case, mode):
    eng, n = case.eng, case.n
    fit = torch.zeros((2, n), dtype=torch.float64, device=eng.device)
    bh = torch.zeros((2, n, 3), dtype=torch.float32, device=eng.device)
    eng.rollout(case.d_table, eng.to_device(case.idx), case.d_theta, case.sigma, case.sizes, case.d_obsn, case.d_rew, case.ps,
                fit[0], fit[1], 1, bh[0], bh[1], mode, act_noise=eng.to_device(case.noise), episodes=case.E)
    eng.sync()
    return fit.cpu().numpy(), bh.cpu().numpy()


# ------------------------------------------------------------------------------------------------ closed loop
def _closed_run(eng, p, d, act):
    """test_gpu_closed_f64's rollout_closed_mlp call with the policy's activation."""
    orig = eng.rollout_closed_mlp
    eng.rollout_closed_mlp = lambda *a, **k: orig(*a, activation=act, **k)
    try:
        return cf._run(eng, p, d)
    finally:
        del eng.rollout_closed_mlp


# (shape, cluster size): a cluster of one CTA (a shape tanh runs on rollout_closed.cu), simple_conf and obj
_CLOSED = [((8, 32, 32, 4), 1), ((15, 256, 256, 3), 2), ((17, 256, 256, 256, 6), 4)]


@pytest.mark.parametrize('noisy', [False, True], ids=['plain', 'noise-E2'])
@pytest.mark.parametrize('shape,C', _CLOSED, ids=[str(c) for _, c in _CLOSED])
@pytest.mark.parametrize('name', list(ACTS))
def test_closed_loop_against_float64(eng, name, shape, C, noisy):
    act, f64act = ACTS[name]
    p = cf.Problem(name, shape, 60, 1.0, 0.5, seed=11 + C, n_pairs=4, E=2 if noisy else 1, ac_std=0.05 if noisy else 0.0)
    assert eng.closed_mlp_plan(list(shape), p.band, activation=act)[0] == C
    d = cf.build(p)
    got = _closed_run(eng, p, d, act)
    assert got[5] == 1                                                        # one launch
    args, kw = cf.truth_args(p, d)
    tr = act_f64.closed_truth(*args, activation=f64act, **kw)
    cf._check(f'{name} {shape}', p, got[:5], tr, d['saved'], d['spec'].pos_scale)
    again = _closed_run(eng, p, d, act)
    assert np.array_equal(got[0], again[0]) and np.array_equal(got[1], again[1]) and np.array_equal(got[4], again[4])
    cf._check(f'{name} {shape} rerun', p, again[:5], tr, d['saved'], d['spec'].pos_scale)   # ObStat: atomics' order


@pytest.mark.parametrize('shape', [(8, 32, 32, 4), (15, 256, 256, 3)])
def test_closed_tanh_through_the_new_entry_point_is_the_old_one(eng, shape):
    p = cf.Problem('tanh', shape, 40, 1.0, 0.5, seed=3, n_pairs=3, E=2, ac_std=0.05)
    d = cf.build(p)
    a, b = _closed_run(eng, p, d, TANH), cf._run(eng, p, d)
    for x, y in zip(a[:2], b[:2]):
        assert np.array_equal(x, y)
    assert eng.closed_mlp_plan(list(shape), p.band, activation=TANH) == eng.closed_mlp_plan(list(shape), p.band)


# ------------------------------------------------------------------------------------------------ generations
def _policies(env, module, n_copies, seed=21):
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    nets = [FeedForward([64, 64], module, env, 0.0) for _ in range(n_copies)]
    P = len(Policy.get_flat(nets[0]))
    rs = np.random.RandomState(seed)
    table = rs.randn(P + 50_000).astype(np.float32)
    theta = (rs.randn(P) * 0.15).astype(np.float32)
    out = []
    for net in nets:
        p = Policy(net, 0.02, Adam(P, 0.01))
        p.flat_params[...] = theta
        p.set_nn_params(p.flat_params)
        out.append(p)
    return out, table


@pytest.mark.parametrize('closed', [False, True], ids=['open', 'closed'])
@pytest.mark.parametrize('name', ['relu', 'elu'])
def test_generations_fused_equal_device_generation_and_python_loop(eng, name, closed):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    from es_pytorch_b200.gym.training_result import RewardResult
    from es_pytorch_b200.nn.obstat import ObStat
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    act, _ = ACTS[name]
    module = {'relu': torch.nn.ReLU(), 'elu': torch.nn.ELU(0.7)}[name]
    obs, nact, T, n = 15, 3, 30, 8
    env = (ClosedLoopEnv if closed else SyntheticEnv)(obs, nact, T)
    (pa, pb, pc), table = _policies(env, module, 3)
    assert pa._module.activation() == act
    nts = [NoiseTable(len(pa), table.copy()) for _ in range(3)]
    streams = [np.random.RandomState(77) for _ in range(3)]
    fused = BatchedRollout(env, T, coins_per_eval=0, fuse_activations=True)
    assert es._can_fuse_step(dist.world(), pa, fused, CenteredRanker())

    def loop(model, use_ac_noise=True):                       # the python loop: the module's own forward at every step
        rews, behv, obsv, steps = run_model(model, env, T, None)
        return RewardResult(rews, behv, obsv, steps)

    pos_a, neg_a, inds_a, _ = es.test_params(dist.world(), n, pa, nts[0], ObStat((obs,), 0), fused, streams[0])
    pos_b, neg_b, inds_b, _ = es.test_params(dist.world(), n, pb, nts[1], ObStat((obs,), 0), loop, streams[1])
    assert np.array_equal(inds_a, inds_b)
    assert np.array_equal(streams[0].get_state()[1], streams[1].get_state()[1]) and streams[0].get_state()[2] == streams[1].get_state()[2]
    fa, fb = np.concatenate((pos_a, neg_a)), np.concatenate((pos_b, neg_b))
    mass = np.abs(fb).max() + 1.0
    assert np.abs(fa - fb).max() <= 1e-5 * mass * T, np.abs(fa - fb).max()
    # the DeviceGeneration this route built is the one es.step queues: same inputs, bit-identical fitness
    gen = fused._gen
    assert gen.activation == act and gen.act_key == act.key()
    again = es.test_params(dist.world(), n, pc, nts[2], ObStat((obs,), 0), fused, streams[2])
    assert np.array_equal(again[0], pos_a) and np.array_equal(again[1], neg_a) and np.array_equal(again[2], inds_a)
    # es.step: one fused generation with its noiseless evaluation, against the same generation queued by hand
    class Cfg(dict):
        __getattr__ = dict.__getitem__
    cfg = Cfg(general=Cfg(policies_per_gen=2 * n, batch_size=500), policy=Cfg(l2coeff=0.005))
    rs_step, rs_ref = np.random.RandomState(5), np.random.RandomState(5)
    (ps, pr), _ = _policies(env, module, 2)
    step_fn = BatchedRollout(env, T, coins_per_eval=0, fuse_activations=True)
    tr, _ = es.step(cfg, dist.world(), ps, NoiseTable(len(ps), table.copy()), env, step_fn, rs_step, CenteredRanker(), Reporter())
    ref_fn = BatchedRollout(env, T, coins_per_eval=0, fuse_activations=True)
    gen = es._device_generation(ref_fn, pr, NoiseTable(len(pr), table.copy()), [rs_ref])
    fp, fn = gen.evaluate(n)
    eng.sync()
    rk = step_fn._gen.fit_local.cpu().numpy()
    assert np.array_equal(rk[0, :, 0], fp.cpu().numpy()[:, 0]) and np.array_equal(rk[1, :, 0], fn.cpu().numpy()[:, 0])
    assert np.array_equal(step_fn._gen.idx.cpu().numpy(), gen.idx.cpu().numpy())
    # the noiseless evaluation of the new theta: the per-call route, one launch with the activation
    assert np.isfinite(tr.result[0])
    want = loop(ps._module).result[0]
    assert abs(tr.result[0] - want) <= 1e-5 * (abs(want) + 1.0) * T, (tr.result[0], want)


def test_binned_relu_stays_unfused_with_the_flag(eng):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
    from es_pytorch_b200.nn.nn import FFBinned
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker
    env = SyntheticEnv(15, 3, 20)
    net = FFBinned([64, 64], torch.nn.ReLU(), env, 5)
    pol = Policy(net, 0.02, Adam(len(Policy.get_flat(net)), 0.01))
    b = BatchedRollout(env, 20, coins_per_eval=0, fuse_activations=True)
    assert not es._can_fuse_step(dist.world(), pol, b, CenteredRanker())
    l0 = eng.launches
    b(net, False)                                                             # the module's own forward
    assert eng.launches == l0
