"""GPU: policies with ReLU, leaky-ReLU, ELU and sigmoid activations (es_rollout_*_activation) against the float64 truth.

* open loop, ES_ROLLOUT_F32 (the general float32 kernel) and ES_ROLLOUT_TC3 (the wide tensor-core kernel's code) at the
  shipped shapes, judged as the tanh kernels are (test_gpu_rollout_f64's EVAL_REL / RMS_BOUND / ACT_ERR against
  f64_rollout's truth with the float64 activation); action noise and episodes, T = 1 and partial tiles, sigma = 0, pair counts
  around the SM count and multi-launch float32 chunks;
* closed loop at clusters of 1, 2 and 4 CTAs against closed_f64.truth with the activation (test_gpu_closed_f64's
  bounds), ObStat sums included;
* launch edges: TC3 around its launch chunk, F32 with 8 ragged layers and around the switch to staged weights (H = 196 ..
  198), the wide kernel's layer shapes (widths 192 and mixed, act 32, obs 1 and 256, four hidden layers), the closed loop in
  clusters of 2 and 8; results independent of the pair order (a reversed run, bit for bit) in F32, TC3 and the closed loop;
* the bounds shown to reject truths with the activation evaluated wrongly (tanh in one layer, no output activation, torch's
  default slope / alpha), and the activations' own regimes in F32 and the closed loop (sigmoid's saturated tails, ELU near 0,
  leaky slopes 0, -0.5 and 3, ELU with alpha 0);
* refusals (ES_ROLLOUT_TC, unknown kinds, a non-finite parameter, obs beyond TC3's coverage) and the float16 guard of TC3,
  which looks at the episode's rows only (not the zero observations that pad the last tile);
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
import f64_rollout as f64  # noqa: E402
from test_gpu_rollout_f64 import ACT_ERR, EVAL_REL, RMS_BOUND, U, Case, _sample  # noqa: E402
import closed_f64  # noqa: E402
import test_gpu_closed_f64 as cf  # noqa: E402
import test_gpu_rollout_f64 as rf  # noqa: E402
import test_gpu_rollout_wide as rw  # noqa: E402

pytestmark = pytest.mark.gpu

F32, TC, TC3 = _lib.ES_ROLLOUT_F32, _lib.ES_ROLLOUT_TC, _lib.ES_ROLLOUT_TC3
ACTS = {
    'relu': (Activation(_lib.ES_ACT_RELU, 0.0), f64.relu),
    'leaky': (Activation(_lib.ES_ACT_LEAKY_RELU, float(np.float32(0.1))), f64.leaky_relu(0.1)),
    'elu': (Activation(_lib.ES_ACT_ELU, float(np.float32(0.7))), f64.elu(0.7)),
    'sigmoid': (Activation(_lib.ES_ACT_SIGMOID, 0.0), f64.sigmoid),
}
TANH = Activation(_lib.ES_ACT_TANH, 0.0)
# rms error over the checked evaluations relative to their fitness spread, about twice the largest value measured on an H100
# 80GB HBM3 (700 W power limit) over this file: F32 3.74e-6 (sigmoid at 376-64-64-17: its fast exponential and division),
# TC3 1.08e-5 (relu at 15-256-256-3: the split operands drop the lo * lo products, ~2^-22 of each, and an unbounded activation
# passes that relative error on at full size where tanh saturates).  Per evaluation the tanh files' EVAL_REL holds as it is
# (largest measured err / mass: F32 9.7e-7, TC3 1.8e-6)
RMS = {F32: 8e-6, TC3: 2.5e-5}
# sigmoid: its fast exponential's absolute error (~1e-7 per action, common to both modes) over the small fitness spread of a
# single bounded action: measured up to 2.69e-5 (F32) and 2.18e-5 (TC3) at 7-192-64-128-1 (with another draw of the inputs
# than test_open_loop_against_float64's, where it is 2.5e-6 / 3.0e-6); about twice that
RMS_SIGMOID = {F32: 6e-5, TC3: 5e-5}


def rms_bound(mode, act):
    """The rms/spread bound of a rollout in ``mode`` of a policy with activation ``act`` (an nn.Activation)."""
    return RMS_SIGMOID[mode] if act is not None and act.kind == _lib.ES_ACT_SIGMOID else RMS[mode]
SHAPES = {'humanoid': [376, 64, 64, 17], 'simple_conf': [15, 256, 256, 3], 'obj': [17, 256, 256, 256, 6],
          'flagrun': [28, 128, 256, 256, 128, 8],
          # test_gpu_rollout_wide.test_wide_layer_shapes': widths of 192 and mixed, act 32, obs 1 and 256, four hidden of 64
          'mixed': [7, 192, 64, 128, 1], 'act32': [9, 128, 128, 32], 'obs1': [1, 64, 128, 4], 'obs256': [256, 256, 64, 5],
          'four-hidden-64': [20, 64, 64, 64, 64, 2]}


class ActCase(Case):
    """test_gpu_rollout_f64's Case for a policy with activation ``name`` (or ``act``: an (Activation, float64 form) pair)."""

    def __init__(self, eng, name, sizes, T, n, seed, act=None, **kw):
        super().__init__(eng, sizes, T, n, seed, **kw)
        self.act, self.f64act = act or (ACTS[name] if name != 'tanh' else (TANH, np.tanh))
        self.launches = None

    def upload(self):
        """After the host arrays were changed in place."""
        d = lambda a: self.eng.to_device(np.ascontiguousarray(a))
        self.d_table, self.d_theta, self.d_obsn, self.d_rew = d(self.table), d(self.theta), d(self.obsn), d(self.rew)

    def run(self, mode, act=None, sigma=None, reverse=False):
        """(fitness [2, n], behaviour [2, n, 3]); ``reverse``: the pairs in reverse order (indices and noise), results
        returned in the original order.  The call's launches in ``self.launches``."""
        eng, n = self.eng, self.n
        sl = slice(None, None, -1) if reverse else slice(None)
        fit = torch.full((2, n), float('nan'), dtype=torch.float64, device=eng.device)
        bh = torch.full((2, n, 3), float('nan'), dtype=torch.float32, device=eng.device)
        nz = None if self.noise is None else eng.to_device(np.ascontiguousarray(self.noise[sl]))
        l0 = eng.launches
        eng.rollout(self.d_table, eng.to_device(np.ascontiguousarray(self.idx[sl])), self.d_theta,
                    self.sigma if sigma is None else sigma, self.sizes, self.d_obsn, self.d_rew, self.ps, fit[0], fit[1], 1, bh[0],
                    bh[1], mode, act_noise=nz, episodes=self.E, activation=self.act if act is None else act)
        eng.sync()
        self.launches = eng.launches - l0
        f, b = fit.cpu().numpy()[:, sl], bh.cpu().numpy()[:, sl]
        assert not np.isnan(f).any() and not np.isnan(b).any(), 'an evaluation was not written'
        return f, b

    def truth(self, pairs, f64act=None):
        """``f64act``: in place of the policy's float64 activation (one function, or a list of one per layer)."""
        return f64.rollout_f64(self.table, self.idx, self.theta, self.sigma, self.sizes, self.obsn, self.rew, self.ps,
                               self.noise, self.E, pairs, activation=self.f64act if f64act is None else f64act)


def _check(tag, mode, case, f, b, pairs, rms_check=True, truth=None):
    tf, tb, mass, mag = case.truth(pairs) if truth is None else truth
    f, b = f[:, pairs], b[:, pairs]
    err = np.abs(f - tf)
    spread = max(tf.std(), 1e-3 * math.sqrt(case.T))
    rms = math.sqrt((err ** 2).mean())
    worst = (err / mass).max()
    bound = rms_bound(mode, case.act)
    print(f'\n[act f64] {tag} mode={mode}: rms/spread {rms / spread:.3g} (bound {bound:.3g}), max err/mass {worst:.3g} '
          f'(bound {EVAL_REL[mode]:.3g})')
    assert np.all(err <= EVAL_REL[mode] * mass), (tag, worst)
    assert not rms_check or rms <= bound * spread, (tag, rms / spread)
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
    a, k = list(ACTS).index(name), list(SHAPES).index(shape)
    # the wide test's shapes (k >= 4) seeded apart: at seed 8 one deep ReLU evaluation has no action above 0 at any step
    case = ActCase(eng, name, sizes, 300, 12, seed=10 * a + k + (700 if k >= 4 else 0))
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


def test_tc3_chunk_edges_and_pair_order(eng):
    """15-256-256-3 in launch chunks of c pairs (test_gpu_rollout_wide._tcw_chunk): c - 1, c and c + 1 pairs, with pairs c - 1, c
    and c + 1 against the truth; every run bit-identical to one with the pairs reversed (no result depends on the grid, the
    chunking or the order of the pairs)."""
    sizes = [15, 256, 256, 3]
    c = rw._tcw_chunk(sizes, TC3)
    for n, name in ((c - 1, 'sigmoid'), (c, 'elu'), (c + 1, 'relu')):
        case = ActCase(eng, name, sizes, 64, n, seed=n, E=2, ac_std=0.05)
        f, b = _run_check(f'{name} n={n} (chunk {c})', case, TC3, pairs=_sample(n, must=(c - 1, c, c + 1), k=10), repeat=False)
        assert case.launches == rw._tcw_launches(sizes, TC3, n)
        fr, br = case.run(TC3, reverse=True)
        assert np.array_equal(f, fr) and np.array_equal(b, br), f'{name} n={n}: the reversed run differs'


def _f32_launches(sizes, n):
    """ES_ROLLOUT_F32 with an activation: the general kernel only (never the packed-FMA one), one launch per chunk, two
    with staged weights."""
    gw, chunk = rf._f32_layout(sizes)
    return 2 * -(-n // chunk) if gw else 1


@pytest.mark.parametrize('sizes', [[15, 256, 256, 3], [17, 64, 64, 6]], ids=['staged', 'shared'])
def test_f32_pair_order(eng, sizes):
    """ES_ROLLOUT_F32 with the weights staged in global memory and in shared memory: the pairs reversed, bit for bit (at
    least SM count / 2 pairs, so that no episode is split over the SMs)."""
    gw = rf._f32_layout(sizes)[0]
    assert gw == (sizes[1] == 256)
    n = eng.sm_count // 2 + 7
    case = ActCase(eng, 'leaky', sizes, 90, n, seed=n, E=2, ac_std=0.05)
    f, b = _run_check(f'leaky F32 n={n}', case, F32, pairs=_sample(n, k=10), repeat=False)
    assert case.launches == _f32_launches(sizes, n) == (2 if gw else 1)
    fr, br = case.run(F32, reverse=True)
    assert np.array_equal(f, fr) and np.array_equal(b, br)


# ES_MAX_LAYERS = 8 ragged layers in shared memory, and 15-H-H-3 around the switch to staged weights (H = 197 / 198)
_F32_SHAPES = [('ragged8', [5, 7, 33, 3, 130, 1, 64, 9, 2], False), ('H196', [15, 196, 196, 3], False),
               ('H197', [15, 197, 197, 3], False), ('H198', [15, 198, 198, 3], True)]


@pytest.mark.parametrize('name', list(ACTS))
@pytest.mark.parametrize('shape,sizes,gw', _F32_SHAPES, ids=[s[0] for s in _F32_SHAPES])
def test_f32_ragged_layers_and_the_staged_weights_switch(eng, shape, sizes, gw, name):
    assert rf._f32_layout(sizes)[0] == gw
    for n in (5, eng.sm_count // 2 + 3):                        # split over the SMs (few pairs) and not
        case = ActCase(eng, name, sizes, 77, n, seed=n + len(sizes), E=2, ac_std=0.05)
        _run_check(f'{name} {shape} n={n}', case, F32, pairs=_sample(n, k=12), repeat=False)
        assert case.launches == _f32_launches(sizes, n)


# ------------------------------------------------------------------------------------------------ the bounds are sensitive
def _mutated_forms(name, which):
    """The policy's float64 activation per layer, evaluated wrongly on purpose (tests/gen_stages.py's modelled bugs)."""
    act, f = ACTS[name]
    if which == 'default_param':
        return {'leaky': f64.leaky_relu(0.01), 'elu': f64.elu(1.0)}[name]
    return lambda n_layers: ([np.tanh] + [f] * (n_layers - 1) if which == 'tanh_layer' else [f] * (n_layers - 1) + [lambda z: z])


@pytest.mark.parametrize('mode,shape', [(F32, 'simple_conf'), (TC3, 'simple_conf'), (F32, 'humanoid')],
                         ids=['F32-simple_conf', 'TC3-simple_conf', 'F32-humanoid'])
@pytest.mark.parametrize('name', list(ACTS))
def test_bounds_reject_mutated_truths(eng, name, mode, shape):
    """_check accepts the device's fitness against the truth and rejects it against each truth with the activation
    evaluated wrongly: tanh in the first hidden layer, no activation after the output layer, and (leaky ReLU, ELU) torch's
    default slope 0.01 / alpha 1.0 in place of the policy's."""
    sizes = SHAPES[shape]
    case = ActCase(eng, name, sizes, 300, 40, seed=3, ac_std=0.01)
    pairs = _sample(40, k=16)
    f, b = case.run(mode)
    truth = case.truth(pairs)
    _check(f'{name} unmutated', mode, case, f, b, pairs, truth=truth)
    whats = ('tanh_layer', 'no_output') + (('default_param',) if name in ('leaky', 'elu') else ())
    for what in whats:
        forms = _mutated_forms(name, what)
        bad = case.truth(pairs, f64act=forms if what == 'default_param' else forms(len(sizes) - 1))
        tf, mass = bad[0], bad[2]
        spread = max(tf.std(), 1e-3 * math.sqrt(case.T))
        fp = f[:, pairs]
        print(f'  mutated {what}: rms/spread {math.sqrt(((fp - tf) ** 2).mean()) / spread:.3g}, '
              f'max err/mass {(np.abs(fp - tf) / mass).max():.3g}')
        with pytest.raises(AssertionError):
            _check(f'{name} mutated {what}', mode, case, f, b, pairs, truth=bad)


# ------------------------------------------------------------------------------------------------ the activations' own regimes
def _place_in_sigmoid_tails(theta, sizes, rs):
    """Every layer's biases moved by +-|z| spread over [0, 100]: pre-activations in sigmoid's saturated tails (where
    __fdividef(1, 1 + __expf(-z)) returns 0 from z below about -87) and through its transition, without scaling any weight
    (a scaled weight would scale the rounding of the products with it)."""
    th = theta.astype(np.float64)
    for _, bo, _, fo in f64.layer_slices(sizes):
        th[bo:bo + fo] += rs.permutation(np.linspace(0.0, 100.0, fo)) * rs.choice([-1.0, 1.0], fo)
    return th.astype(np.float32)


# name -> (Activation, float64 form, how theta and the table are changed: 'tails' (_place_in_sigmoid_tails), 'small' (theta,
# the noise table and the action noise times SMALL: ELU's pre-activations within |z| < 1e-3, where exp(z) - 1 would lose every
# digit) or None)
SMALL = np.float32(3e-4)
REGIMES = {
    'sigmoid_tails': (Activation(_lib.ES_ACT_SIGMOID, 0.0), f64.sigmoid, 'tails'),
    'elu_near_zero': (ACTS['elu'][0], ACTS['elu'][1], 'small'),
    'leaky_slope_0': (Activation(_lib.ES_ACT_LEAKY_RELU, 0.0), f64.leaky_relu(0.0), None),
    'leaky_slope_-0.5': (Activation(_lib.ES_ACT_LEAKY_RELU, -0.5), f64.leaky_relu(-0.5), None),
    'leaky_slope_3': (Activation(_lib.ES_ACT_LEAKY_RELU, 3.0), f64.leaky_relu(3.0), None),
    'elu_alpha_0': (Activation(_lib.ES_ACT_ELU, 0.0), f64.elu(0.0), None),
}


def _regime_premise(regime, z):
    """The pre-activations ``z`` (float64, every layer) reach the regime."""
    if regime == 'sigmoid_tails':
        assert z.max() > 80 and z.min() < -88 and (np.abs(z) < 2).any()
    elif regime == 'elu_near_zero':
        assert np.abs(z).max() < 1e-3 and (z < 0).mean() > 0.2
    else:
        assert (z < 0).mean() > 0.2 and (z > 0).mean() > 0.2


@pytest.mark.parametrize('regime', list(REGIMES))
def test_f32_activation_regimes(eng, regime):
    act, form, how = REGIMES[regime]
    sizes = [17, 64, 64, 6]
    case = ActCase(eng, None, sizes, 200, 24, seed=31, act=(act, form), E=2, ac_std=0.05)
    rs = np.random.RandomState(32)
    if how == 'tails':
        case.theta = _place_in_sigmoid_tails(case.theta, sizes, rs)
    elif how == 'small':
        case.theta = (case.theta * SMALL).astype(np.float32)
        case.table = (case.table * SMALL).astype(np.float32)
        case.noise = (case.noise * SMALL).astype(np.float32)
    case.upload()
    zs, h = [], case.obsn.astype(np.float64)
    for k in (0, case.n - 1):
        w = f64.perturbed(case.table, case.idx[k], case.theta, case.sigma, 1.0)
        h = case.obsn.astype(np.float64)
        for wo, bo, fi, fo in f64.layer_slices(sizes):
            z = h @ w[wo:wo + fi * fo].reshape(fo, fi).T + w[bo:bo + fo]
            zs.append(z.ravel())
            h = form(z)
    _regime_premise(regime, np.concatenate(zs))
    _run_check(f'F32 {regime}', case, F32)


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


def test_tc3_guard_looks_at_the_episode_rows_only(eng):
    """A ReLU policy whose forward of a zero observation leaves float16 range while every step of the episode stays inside:
    observation column 0 held at 5; layer 1's first 128 units with bias +B, cancelled exactly on every live row by weights
    -B / 5 on that column (their other weights 0), the other 128 units as drawn; layer 2's weights 1 + theta's; sigma 0.  The
    rows of the last tile beyond T (zero observations) reach ~128 B in layer 2; TC3 must not flag them, and agrees with F32
    and the float64 truth."""
    B, sizes, T = 1000.0, [15, 256, 256, 3], 100                  # T = 100: rows 100 .. 127 of the tile are padding
    case = ActCase(eng, 'relu', sizes, T, 4, seed=12)
    case.sigma = 0.0
    case.obsn[:, 0] = 5.0
    th = case.theta.copy()
    (w1, b1, fi1, fo1), (w2, b2, fi2, fo2), _ = f64.layer_slices(sizes)
    W1 = th[w1:w1 + fi1 * fo1].reshape(fo1, fi1)
    W1[:128] = 0.0
    W1[:128, 0] = -B / 5
    th[b1:b1 + 128] = B
    th[w2:w2 + fi2 * fo2] += 1.0
    case.theta = th
    case.upload()
    # the premise, in float64: padded rows beyond float16 range in layer 2, every live row within it
    for x in (case.obsn.astype(np.float64), np.zeros((1, sizes[0]))):
        h = x
        for wo, bo, fi, fo in f64.layer_slices(sizes)[:2]:
            h = np.maximum(h @ th[wo:wo + fi * fo].reshape(fo, fi).T.astype(np.float64) + th[bo:bo + fo], 0.0)
        if x.shape[0] == 1:
            assert np.abs(h).max() > 65504
        else:
            assert np.abs(h).max() < 65504 / 4
    f3, b3 = case.run(TC3)
    assert eng.lib.es_check_async(eng._ctx) == 0
    # (per evaluation only: sigma = 0 leaves every evaluation the same policy, no spread to measure the rms against)
    _check('relu padded rows TC3', TC3, case, f3, b3, list(range(case.n)), rms_check=False)
    f, b = case.run(F32)
    _check('relu padded rows F32', F32, case, f, b, list(range(case.n)), rms_check=False)
    tf, _, mass, _ = case.truth(list(range(case.n)))
    assert np.all(np.abs(f3 - f) <= 2 * EVAL_REL[TC3] * mass)


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
    tr = closed_f64.truth(*args, activation=f64act, **kw)
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


def _reversed(p, d):
    """Problem ``p``'s inputs with the pairs in reverse order (indices, noise and the saved evaluations)."""
    n = p.n_pairs
    return dict(d, idx=d['idx'][::-1].copy(), noise=None if d['noise'] is None else d['noise'][::-1].copy(),
                saved=[(n - 1 - k, s) for k, s in d['saved']])


# (shape, band, cluster size, T): simple_conf, and test_gpu_closed_f64's eight-CTA shape (band 16)
_CLOSED_ORDER = [((15, 256, 256, 3), 8, 2, 60), ((384, 256, 256, cf.largest_eight_cta_width(), 64), 16, 8, 12)]


@pytest.mark.parametrize('name', list(ACTS))
@pytest.mark.parametrize('shape,band,C,T', _CLOSED_ORDER, ids=[f'C{c}' for _, _, c, _ in _CLOSED_ORDER])
def test_closed_loop_clusters_and_pair_order(eng, name, shape, band, C, T):
    """Against the float64 truth at clusters of 2 and 8 CTAs, with action noise and 2 episodes; the pairs reversed give
    every fitness and behaviour bit for bit (the ObStat sums: within the truth's bound, their atomics have no fixed order)."""
    act, f64act = ACTS[name]
    p = cf.Problem(name, shape, T, 1.0, 0.5, seed=7 + C, band=band, n_pairs=3, E=2, ac_std=0.05)
    assert closed_f64.cluster_size(list(shape), band) == C and eng.closed_mlp_plan(list(shape), band, activation=act)[0] == C
    d = cf.build(p)
    got = _closed_run(eng, p, d, act)
    assert got[5] == 1
    args, kw = cf.truth_args(p, d)
    tr = closed_f64.truth(*args, activation=f64act, **kw)
    cf._check(f'{name} {shape}', p, got[:5], tr, d['saved'], d['spec'].pos_scale)
    rev = _closed_run(eng, p, _reversed(p, d), act)
    assert np.array_equal(got[0], rev[0][:, ::-1]) and np.array_equal(got[1], rev[1][:, ::-1]), 'the reversed run differs'
    cf._check(f'{name} {shape} reversed', p, (rev[0][:, ::-1], rev[1][:, ::-1]) + rev[2:5], tr, d['saved'], d['spec'].pos_scale)


@pytest.mark.parametrize('regime', list(REGIMES))
def test_closed_loop_activation_regimes(eng, regime):
    """REGIMES in the closed loop (a cluster of one CTA), with action noise; the loop shown not to amplify rounding first
    (closed_f64.growth <= 100, as test_gpu_closed_f64's problems)."""
    act, form, how = REGIMES[regime]
    p = cf.Problem(regime, (8, 32, 32, 4), 60, 1.0, 0.2, seed=41, n_pairs=4, E=2, ac_std=0.05)
    d = cf.build(p)
    if how == 'tails':
        d['theta'] = _place_in_sigmoid_tails(d['theta'], list(p.sizes), np.random.RandomState(42))
    elif how == 'small':
        d['theta'] = (d['theta'] * SMALL).astype(np.float32)
        d['table'] = (d['table'] * SMALL).astype(np.float32)
        d['noise'] = (d['noise'] * SMALL).astype(np.float32)
    args, kw = cf.truth_args(p, d)
    growth = closed_f64.growth(*args, activation=form, **kw)
    assert growth <= 100, growth
    got = _closed_run(eng, p, d, act)
    tr = closed_f64.truth(*args, activation=form, **kw)
    cf._check(f'closed {regime} (growth {growth:.3g})', p, got[:5], tr, d['saved'], d['spec'].pos_scale)


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
