"""Every open-loop rollout mode against the float64 reference (tests/f64_rollout.py), at the shipped configs' policies and
at the launch, tile and dispatch edges of each kernel.

One assert helper (``_check``) judges every case:
* per evaluation ``|f - truth| <= EVAL_REL * mass`` -- 1e-5 (the suite's float32 bound) for ES_ROLLOUT_F32 and
  ES_ROLLOUT_TC3, the looser class of the single-float16 ES_ROLLOUT_TC otherwise.  The mass is
  ``sum_t sum_j |a_tj c_tj|``, not ``sum_t |r_t|``: the error of a step's reward is that of a dot product, relative to the
  sum of its products' magnitudes.  The two agree on long episodes, but one step can earn ~0 from large products, and at
  T = 1 a correct split tensor-core rollout measured 3e-5 of ``|r|`` and the float32 floor of a dot product is
  ``act * 2^-24`` of the products;
* over the checked evaluations ``rms(f - truth) <= RMS_BOUND * spread`` (spread = the truth's standard deviation, floored at
  1e-3 sqrt(T) as in test_gpu_kernels.py), each bound about 2x the largest value measured on an H100 SXM (80 GB);
* final positions within float32 rounding of their T-term sums (2^-24 times the reference's position magnitude, twice) plus
  the actions' own error over T steps.
``test_bounds_reject_mutated_truths`` shows that these bounds reject a truth with the last step's reward dropped, with one
layer's bias unperturbed and with the signs of one pair swapped (measured: 0.04 .. 0.36 of the spread rms, where the bounds
are 3e-6 .. 5e-3).

Which kernel and how many launches a case takes is restated from the host launchers (``_f32_layout``, ``_f32x_fits``) and
asserted through ``Engine.launches``, so a change of the launch layout fails here instead of moving a case to another path.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib
from oracle import es_oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import f64_rollout as f64  # noqa: E402

pytestmark = pytest.mark.gpu

F32, TC, TC3 = _lib.ES_ROLLOUT_F32, _lib.ES_ROLLOUT_TC, _lib.ES_ROLLOUT_TC3
U = 2.0 ** -24
SMEM = 227 * 1024
# per-evaluation bound relative to the reward mass.  Largest values measured on an H100 SXM (80 GB, 400 W power limit) over
# this file: F32 1.8e-7, TC3 1.7e-6 (both at T = 1), TC 4.4e-4 (T = 1)
EVAL_REL = {F32: 1e-5, TC3: 1e-5, TC: 1e-3}
# rms error over the checked evaluations relative to their fitness spread.  Largest values measured there: F32 1.45e-6
# (28-256-256-256-8, four launches), TC3 4.1e-6 (act 31), TC 2.3e-3 (T = 128)
RMS_BOUND = {F32: 3e-6, TC3: 8e-6, TC: 5e-3}
# error of one action, for the position bound: float32 arithmetic / float16 products
ACT_ERR = {F32: 1e-5, TC3: 1e-5, TC: 3e-3}


# ---------------------------------------------------------------------------------------------- the launchers, restated
def _r4(x):
    return (x + 3) & ~3


def _f32_layout(sizes):
    """rollout_f32.cu's es_impl_rollout_f32: (weights staged in global memory (GW), pairs per launch)."""
    soff = xmax = 0
    for fi, fo in zip(sizes[:-1], sizes[1:]):
        in4 = _r4(fi)
        pitch = in4 if (in4 >> 2) & 1 else in4 + 4
        soff += fo * pitch
        xmax = max(xmax, in4, _r4(fo))
    soff += sum(_r4(fo) for fo in sizes[1:])
    w_floats = _r4(soff)
    act_smem = 2 * 32 * xmax * 4 + 32 * 8
    gw = w_floats * 4 + act_smem > SMEM
    return gw, (max(1, (256 << 20) // (2 * w_floats * 4)) if gw else None)


def _f32x_fits(obs, act):
    """rollout_f32x.cu's fx_layout(obs, act).total <= 227 KB."""
    nkc, act4 = -(-obs // 16), _r4(act)
    total = (64 * (nkc * 16 + 4) * 4 + 6 * 128 * 16 * 4 + 128 * 64 * 4 + 2 * 64 * 68 * 4 + 2 * act4 * 68 * 4
             + (2 * 96 + 64) * 4 + 128 * 16 + 16 * 16 + 32 + 2 * 6 * 8)
    return total <= SMEM


def _uses_f32x(sizes, n, sm):
    return (len(sizes) == 4 and sizes[1] == sizes[2] == 64 and sizes[3] <= 32 and 2 * n >= sm
            and _f32x_fits(sizes[0], sizes[3]))


def _f32_launches(sizes, n, sm):
    """Launches of one F32 rollout: packed-FMA = prep + ubase + kernel; general = one per chunk, two with staged weights."""
    if _uses_f32x(sizes, n, sm):
        return 3
    gw, chunk = _f32_layout(sizes)
    return 2 * -(-n // chunk) if gw else 1


def _chunks(sizes, n):
    gw, chunk = _f32_layout(sizes)
    chunk = chunk if gw else n
    return [(p0, min(chunk, n - p0)) for p0 in range(0, n, chunk)]


# ---------------------------------------------------------------------------------------------- cases
class Case:
    """Seeded inputs of one rollout, on the host and on the device."""

    def __init__(self, eng, sizes, T, n, seed, E=1, ac_std=0.0, L=None, idx=None):
        rs = np.random.RandomState(seed)
        self.eng, self.sizes, self.T, self.n, self.E = eng, list(sizes), T, n, E
        self.P = f64.n_params(sizes)
        self.L = L or self.P + 300_000
        self.table = rs.randn(self.L).astype(np.float32)
        self.theta = (rs.randn(self.P) * 0.1).astype(np.float32)
        self.idx = rs.randint(0, self.L - self.P, size=n).astype(np.int64) if idx is None else np.asarray(idx, np.int64)
        self.idx[0], self.idx[-1] = 0, self.L - self.P - 1
        self.obsn = np.clip(rs.randn(T, sizes[0]), -5, 5).astype(np.float32)
        self.rew = rs.randn(T, sizes[-1]).astype(np.float32)
        self.noise = (rs.randn(n, 2, E, T, sizes[-1]) * ac_std).astype(np.float32) if ac_std else None
        self.sigma, self.ps = 0.02, 0.05
        d = lambda a: eng.to_device(np.ascontiguousarray(a))
        self.d_table, self.d_theta, self.d_obsn, self.d_rew = d(self.table), d(self.theta), d(self.obsn), d(self.rew)

    def run(self, mode, fit_stride=1, behv=True, reverse=False):
        """(fitness [2, n], behaviour [2, n, 3] or None, launches).  ``reverse``: the pairs in reverse order (indices and
        noise), results returned in the original order."""
        eng, n = self.eng, self.n
        sl = slice(None, None, -1) if reverse else slice(None)
        idx = self.eng.to_device(np.ascontiguousarray(self.idx[sl]))
        nz = None if self.noise is None else self.eng.to_device(np.ascontiguousarray(self.noise[sl]))
        fit = torch.full((2, n * fit_stride), float('nan'), dtype=torch.float64, device=eng.device)
        bh = torch.full((2, n, 3), float('nan'), dtype=torch.float32, device=eng.device) if behv else None
        l0 = eng.launches
        eng.rollout(self.d_table, idx, self.d_theta, self.sigma, self.sizes, self.d_obsn, self.d_rew, self.ps, fit[0], fit[1],
                    fit_stride, None if bh is None else bh[0], None if bh is None else bh[1], mode, act_noise=nz,
                    episodes=self.E)
        eng.sync()
        launches = eng.launches - l0
        f = fit.cpu().numpy()
        if fit_stride > 1:                                   # the other columns (novelty in the NSRA layout) are untouched
            assert np.isnan(f.reshape(2, n, fit_stride)[:, :, 1:]).all()
        f = f[:, ::fit_stride]
        b = None if bh is None else bh.cpu().numpy()
        if reverse:
            f, b = f[:, ::-1], None if b is None else b[:, ::-1]
        assert not np.isnan(f).any() and (b is None or not np.isnan(b).any()), 'an evaluation was not written'
        return f, b, launches

    def truth(self, pairs):
        return f64.rollout_f64(self.table, self.idx, self.theta, self.sigma, self.sizes, self.obsn, self.rew, self.ps,
                               self.noise, self.E, pairs)


def _sample(n, must=(), k=24, seed=0):
    """``must`` (clipped to [0, n)) plus random pairs up to k, sorted."""
    s = {p for p in must if 0 <= p < n} | {0, n - 1}
    rest = np.random.RandomState(seed).permutation(n)
    for p in rest:
        if len(s) >= k:
            break
        s.add(int(p))
    return sorted(s)


def _check(tag, mode, case, f, b, pairs, truth):
    """The one assert helper: f, b are the device's [2, len(pairs)] / [2, len(pairs), 3] values of ``pairs``."""
    tf, tb, mass, mag = truth
    err = np.abs(f - tf)
    spread = max(tf.std(), 1e-3 * math.sqrt(case.T))
    rms = math.sqrt((err ** 2).mean())
    worst = (err / mass).max()
    print(f'\n[f64] {tag} mode={mode}: rms/spread {rms / spread:.3g} (bound {RMS_BOUND[mode]:.3g}), '
          f'max err/mass {worst:.3g} (bound {EVAL_REL[mode]:.3g})')
    assert np.all(err <= EVAL_REL[mode] * mass), (tag, worst)
    assert rms <= RMS_BOUND[mode] * spread, (tag, rms / spread)
    if b is not None:
        tol = 2 * U * mag + ACT_ERR[mode] * case.ps * case.T
        assert np.all(np.abs(b - tb) <= tol), (tag, np.abs(b - tb).max())


def _run_and_check(tag, case, mode, pairs, launches=None, **kw):
    f, b, nl = case.run(mode, **kw)
    if launches is not None:
        assert nl == launches, (tag, nl, launches)
    _check(tag, mode, case, f[:, pairs], None if b is None else b[:, pairs], pairs, case.truth(pairs))
    return f, b


# ---------------------------------------------------------------------------------------------- A. staged weights, shipped shapes
_A = [
    # (name, sizes, T, E, n_pairs as a function of the chunk, fit_stride, behv)
    ('nsra: chunk + 1, last launch 1 pair time-split', [15, 256, 256, 3], 2000, 1, lambda c: c + 1, 2, True),
    ('simple_conf: one launch', [15, 256, 256, 3], 2000, 1, lambda c: 100, 2, True),
    ('obj: exact multiple of the chunk', [26, 256, 256, 256, 6], 1000, 1, lambda c: 2 * c, 1, False),
    ('obj-8: four launches', [28, 256, 256, 256, 8], 200, 1, lambda c: 3 * c + 2, 1, True),
    ('flagrun: 10 episodes, 2 chunks + 1', [28, 128, 256, 256, 128, 8], 500, 10, lambda c: 2 * c + 1, 1, True),
    ('ns: T = 10000, three pairs', [26, 256, 256, 256, 6], 10000, 1, lambda c: 3, 1, True),
]


@pytest.mark.parametrize('name,sizes,T,E,npairs,fit_stride,behv', _A, ids=[a[0].split(':')[0] for a in _A])
def test_staged_weights_at_the_shipped_shapes(eng, name, sizes, T, E, npairs, fit_stride, behv):
    """ES_ROLLOUT_F32 with the weights staged in global memory (GW), chunked into launches of <= 256 MiB of weights, with
    action noise (ac_std 0.01 as in the shipped configs).  Every pair at each chunk boundary (p0 - 1, p0, p0 + 1), the first
    and the last pair against the float64 truth; all pairs through a second run with the pairs reversed, bit-identical
    wherever neither run splits that pair's episode over the SMs."""
    sm = eng.sm_count
    gw, chunk = _f32_layout(sizes)
    assert gw
    n = npairs(chunk)
    case = Case(eng, sizes, T, n, seed=sum(sizes) + T, E=E, ac_std=0.01)
    chunks = _chunks(sizes, n)
    bounds = [q for p0, _ in chunks[1:] for q in (p0 - 1, p0, p0 + 1)]
    pairs = _sample(n, bounds, k=max(12, len(bounds) + 3), seed=T)
    f, b = _run_and_check(name, case, F32, pairs, launches=_f32_launches(sizes, n, sm), fit_stride=fit_stride, behv=behv)
    fr, br, _ = case.run(F32, fit_stride=fit_stride, behv=behv, reverse=True)
    split = np.zeros(n, dtype=bool)
    for p0, np_ in chunks:
        split[p0:p0 + np_] |= 2 * np_ < sm
    keep = ~(split | split[::-1])
    assert np.array_equal(f[:, keep], fr[:, keep])
    if behv:
        assert np.array_equal(b[:, keep], br[:, keep])


# ---------------------------------------------------------------------------------------------- B. general kernel
def test_general_kernel_eight_ragged_layers(eng):
    """ES_MAX_LAYERS = 8 layers of widths that are not multiples of 4 (the zeroed padding columns feed the next layer), in
    shared memory, split over the SMs (few pairs) and not; action noise with 2 episodes."""
    sizes = [5, 7, 33, 3, 130, 1, 64, 9, 2]
    assert not _f32_layout(sizes)[0]
    sm = eng.sm_count
    for n in (5, sm):
        case = Case(eng, sizes, 77, n, seed=n, E=2, ac_std=0.05)
        _run_and_check(f'8 layers, {n} pairs', case, F32, _sample(n, k=16), launches=1)


def test_nine_layers_are_refused(eng):
    from es_pytorch_b200._lib import EsLibraryError
    sizes = [5, 4, 4, 4, 4, 4, 4, 4, 4, 2]
    P = f64.n_params(sizes)
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=eng.device)
    fit = torch.zeros(2, 1, dtype=torch.float64, device=eng.device)
    with pytest.raises(EsLibraryError, match='n_layers must be in'):
        eng.rollout(z(P + 10), torch.zeros(1, dtype=torch.int64, device=eng.device), z(P), 0.02, sizes, z(8, 5), z(8, 2), 0.05,
                    fit[0], fit[1])


@pytest.mark.parametrize('H', [192, 196, 197, 198, 200])
def test_shared_memory_to_staged_weights_switch(eng, H):
    """15-H-H-3: the weights leave shared memory for the global scratch between H = 197 and 198 (the restated layout;
    one launch in shared memory, two with staged weights)."""
    assert [_f32_layout([15, h, h, 3])[0] for h in (192, 196, 197, 198, 200)] == [False, False, False, True, True]
    n = eng.sm_count // 2 + 3
    case = Case(eng, [15, H, H, 3], 64, n, seed=H)
    _run_and_check(f'15-{H}-{H}-3', case, F32, _sample(n, k=12), launches=_f32_launches(case.sizes, n, eng.sm_count))


# ---------------------------------------------------------------------------------------------- C. packed-FMA dispatch
@pytest.mark.parametrize('dn', [-1, 0, 1, 'sm', 'sm+1'])
def test_packed_fma_pair_count_edge(eng, dn):
    """2 n_pairs against the SM count: below, the general kernel (one launch, time-split); from there on the packed-FMA
    kernel (prep + ubase + kernel), with one or two pairs per CTA around n_pairs = SM count."""
    sm = eng.sm_count
    n = {'sm': sm, 'sm+1': sm + 1}.get(dn) or -(-sm // 2) + dn
    sizes = [17, 64, 64, 6]
    assert _uses_f32x(sizes, n, sm) == (2 * n >= sm)
    case = Case(eng, sizes, 200, n, seed=n)
    _run_and_check(f'f32x n={n}', case, F32, _sample(n, k=24), launches=_f32_launches(sizes, n, sm))


@pytest.mark.parametrize('obs,act,fits', [(384, 17, True), (385, 17, False), (352, 32, True), (353, 32, False)])
def test_packed_fma_shared_memory_edge(eng, obs, act, fits):
    """The packed-FMA kernel's layout fits up to obs 384 (act <= 20) / 352 (act 32); above, the general kernel runs."""
    assert _f32x_fits(obs, act) == fits
    sm = eng.sm_count
    case = Case(eng, [obs, 64, 64, act], 129, sm, seed=obs + act)
    _run_and_check(f'f32x obs={obs} act={act}', case, F32, _sample(sm, k=24), launches=3 if fits else 1)


@pytest.mark.parametrize('T,E', [(1, 1), (257, 4)])
def test_packed_fma_partial_tiles_with_noise(eng, T, E):
    sm = eng.sm_count
    case = Case(eng, [24, 64, 64, 9], T, sm + 5, seed=T, E=E, ac_std=0.05)
    _run_and_check(f'f32x T={T} E={E}', case, F32, _sample(sm + 5, k=24), launches=3)


# ---------------------------------------------------------------------------------------------- D. tensor cores
_MODES = [pytest.param(TC3, id='tc3'), pytest.param(TC, id='tc')]


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('T', [1, 63, 64, 65, 127, 128, 129])
def test_tc_episode_lengths(eng, mode, T):
    """T < 64 leaves the second consumer warpgroup without live rows; 65 / 127 / 129 end inside a tile."""
    case = Case(eng, [24, 64, 64, 6], T, 9, seed=T)
    _run_and_check(f'tc T={T}', case, mode, list(range(9)))


@pytest.mark.parametrize('mode,obs', [(m, o) for m in (TC3, TC) for o in (7, 8, 63, 64, 376, 383)]
                         + [(TC, 504), (TC, 511)])
def test_tc_observation_sizes(eng, mode, obs):
    """Up to the largest obs whose layout fits in shared memory: 383 (TC3, 6 K chunks) and 511 (TC, 8 K chunks)."""
    case = Case(eng, [obs, 64, 64, 17], 130, 20, seed=obs)
    _run_and_check(f'tc obs={obs}', case, mode, list(range(20)))


@pytest.mark.parametrize('mode,obs', [(TC3, 384), (TC, 512)])
def test_tc_refuses_observations_beyond_shared_memory(eng, mode, obs):
    from es_pytorch_b200._lib import EsLibraryError
    sizes = [obs, 64, 64, 6]
    P = f64.n_params(sizes)
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=eng.device)
    fit = torch.zeros(2, 1, dtype=torch.float64, device=eng.device)
    with pytest.raises(EsLibraryError, match=f'shared memory.*obs_dim <= {obs - 1}'):
        eng.rollout(z(P + 10), torch.zeros(1, dtype=torch.int64, device=eng.device), z(P), 0.02, sizes, z(8, obs), z(8, 6),
                    0.05, fit[0], fit[1], mode=mode)
    small = [obs, 64, 6]                                  # one hidden layer: not a shape of the tensor-core path
    Ps = f64.n_params(small)
    with pytest.raises(EsLibraryError, match=rf'obs\(<={obs - 1}\)-64-64-act\(<=32\)'):
        eng.rollout(z(Ps + 10), torch.zeros(1, dtype=torch.int64, device=eng.device), z(Ps), 0.02, small, z(8, obs), z(8, 6),
                    0.05, fit[0], fit[1], mode=mode)


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('act', [1, 16, 17, 31, 32])
def test_tc_action_sizes_with_tma_shadows(eng, mode, act):
    case = Case(eng, [64, 64, 64, act], 200, 12, seed=act)
    _run_and_check(f'tc act={act}', case, mode, list(range(12)))


@pytest.mark.parametrize('mode', _MODES)
def test_tc_last_slices_of_every_shadow_residue(eng, mode):
    """idx = L - P - 1 - r for r = 0..7: the last admissible slice in each of the 8 shifted shadow copies, with a table
    length that is not a multiple of 8."""
    sizes = [64, 64, 64, 6]
    P = f64.n_params(sizes)
    L = P + 100_003
    assert L % 8 != 0
    idx = [L - P - 1 - r for r in range(8)] + [0, 5, 77, 1001]
    case = Case(eng, sizes, 150, len(idx), seed=8, L=L, idx=idx)
    _run_and_check('tc last slices', case, mode, list(range(len(idx))))


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('which', ['sm-1', 'sm', '2sm+1'])
def test_tc_pair_counts_around_the_sm_count(eng, mode, which):
    sm = eng.sm_count
    n = {'sm-1': sm - 1, 'sm': sm, '2sm+1': 2 * sm + 1}[which]
    case = Case(eng, [24, 64, 64, 6], 150, n, seed=n)
    _run_and_check(f'tc n={n}', case, mode, _sample(n, [sm - 1, sm, 2 * sm], k=24))


@pytest.mark.parametrize('mode', _MODES)
@pytest.mark.parametrize('ac_std,E', [(0.0, 1), (0.05, 1), (0.05, 4)])
def test_tc_action_noise_and_episodes(eng, mode, ac_std, E):
    sm = eng.sm_count
    case = Case(eng, [64, 64, 64, 17], 150, sm + 3, seed=E + int(ac_std * 100), E=E, ac_std=ac_std)
    _run_and_check(f'tc noise={ac_std} E={E}', case, mode, _sample(sm + 3, k=24))


# ---------------------------------------------------------------------------------------------- the bounds are sensitive
def _mutated(case, pairs, what):
    """The float64 truth of ``pairs`` computed wrongly on purpose."""
    fit = np.zeros((2, len(pairs)))
    wo, bo, fi, fo = f64.layer_slices(case.sizes)[0]
    for n, k in enumerate(pairs):
        for s, sign in enumerate((1.0, -1.0)):
            if what == 'sign' and n == 0:
                sign = -sign
            w = f64.perturbed(case.table, case.idx[k], case.theta, case.sigma, sign)
            if what == 'bias':
                w[bo:bo + fo] = case.theta[bo:bo + fo]
            nz = None if case.noise is None else case.noise[k, s].reshape(case.E, case.T, -1)
            r, _, _, _ = f64.episode(w, case.sizes, case.obsn, case.rew, case.ps, nz)
            fit[s, n] = r[:-1].sum() if what == 'last_step' else r.sum()
    return fit


@pytest.mark.parametrize('mode,sizes', [(F32, [15, 256, 256, 3]), (F32, [376, 64, 64, 17]), (TC3, [376, 64, 64, 17]),
                                        (TC, [376, 64, 64, 17])])
def test_bounds_reject_mutated_truths(eng, mode, sizes):
    """_check accepts the device's fitness against the truth and rejects it against each broken truth."""
    case = Case(eng, sizes, 300, 40, seed=3, ac_std=0.01)
    pairs = _sample(40, k=16)
    f, b, _ = case.run(mode)
    f, b = f[:, pairs], b[:, pairs]
    truth = case.truth(pairs)
    _check('unmutated', mode, case, f, b, pairs, truth)
    for what in ('last_step', 'bias', 'sign'):
        bad = (_mutated(case, pairs, what),) + truth[1:]
        with pytest.raises(AssertionError):
            _check(f'mutated {what}', mode, case, f, b, pairs, bad)


# ---------------------------------------------------------------------------------------------- E. one generation at obj.json
def test_device_generation_at_the_obj_config(eng):
    """configs/obj.json's policy and population: 26-256-256-256-6, 320 pairs from 2 streams, T = 1000, ac_std = 0.01, one
    save_obs coin per evaluation, the default F32 rollout (two launches of staged weights).  Indices, coins and stream state
    bit for bit with numpy, the action noise to the last bit of float32, fitness against the float64 truth on a sample,
    rank weights and theta against oracle.es_oracle run on the device's fitness.  (SGD: Adam's first step is
    lr * g / (|g| + 3e-7), which turns float32 summation-order differences of near-zero gradient entries -- 140 038 of
    them here -- into changes of theta far above any float32 tolerance.)"""
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import SGD
    sizes, T, n_per, seeds, ac_std = [26, 256, 256, 256, 6], 1000, 160, (31, 32), 0.01
    P = f64.n_params(sizes)
    rs = np.random.RandomState(26)
    L = P + 2_000_000
    table, theta = rs.randn(L).astype(np.float32), (rs.randn(P) * 0.1).astype(np.float32)
    env = orc.SyntheticEnvSpec(26, 6, T)
    gen = DeviceGeneration(eng.to_device(table), eng.to_device(theta.copy()), sizes, eng.to_device(env.obs_stream),
                           eng.to_device(env.rew_vec), [np.random.RandomState(s) for s in seeds], 0.02, 0.005, SGD(P, 0.01),
                           coins_per_eval=1, save_obs_chance=0.01, pos_scale=env.pos_scale, engine=eng, ac_std=ac_std)
    fpos, fneg = gen.evaluate(n_per)
    eng.sync()
    n = 2 * n_per
    # numpy's streams in the reference's program order: per pair randint, per evaluation the coin and T x act gaussians
    ref_idx, ref_words, ref_noise, streams = [], [], [], [np.random.RandomState(s) for s in seeds]
    for s in streams:
        for _ in range(n_per):
            ref_idx.append(int(s.randint(0, L - P)))
            for _sgn in range(2):
                ref_words += [int.from_bytes(s.bytes(4), 'little') for _ in range(2)]
                ref_noise.append((s.randn(T * 6) * ac_std).astype(np.float32))
    idx = gen.idx.cpu().numpy()
    assert np.array_equal(idx, np.array(ref_idx))
    assert np.array_equal(gen.extras.cpu().numpy().view(np.uint32).reshape(-1), np.array(ref_words, dtype=np.uint32))
    noise = gen.act_noise.cpu().numpy()
    want = np.stack(ref_noise).reshape(noise.shape)
    assert np.abs(noise - want).max() <= np.spacing(np.float32(np.abs(want).max()))
    for a, b in zip(gen.rank_states(), streams):
        sa, sb = a.get_state(), b.get_state()
        assert np.array_equal(sa[1], sb[1]) and sa[2:4] == sb[2:4] and abs(sa[4] - sb[4]) <= 2 * np.spacing(abs(sb[4]))
    # the rollout on the generation's inputs: two launches of staged weights per chunk, the generation's values bit for bit
    fp, fn = fpos.cpu().numpy()[:, 0], fneg.cpu().numpy()[:, 0]
    assert _f32_launches(sizes, n, eng.sm_count) == 4
    fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
    l0 = eng.launches
    eng.rollout(gen.table, gen.idx, gen.theta, 0.02, sizes, gen.obsn, gen.rew_vec, env.pos_scale, fit[0], fit[1],
                act_noise=gen.act_noise)
    eng.sync()
    assert eng.launches - l0 == 4
    assert np.array_equal(fit.cpu().numpy(), np.stack([fp, fn]))
    # fitness against the float64 truth: both chunks' edges and a sample
    case = Case.__new__(Case)
    case.sizes, case.T, case.n, case.E, case.P, case.L = sizes, T, n, 1, P, L
    case.table, case.theta, case.idx, case.sigma, case.ps = table, theta, idx, 0.02, env.pos_scale
    case.obsn = orc.normalise_obs(env.obs_stream[:T], np.zeros(26), np.ones(26), 5.0)
    case.rew, case.noise = env.rew_vec, noise.reshape(n, 2, 1, T, 6)
    chunk = _f32_layout(sizes)[1]
    pairs = _sample(n, [chunk - 1, chunk, chunk + 1], k=16)
    _check('obj generation', F32, case, np.stack([fp, fn])[:, pairs], None, pairs, case.truth(pairs))
    # rank weights and theta: the oracle's ranker and Adam step on the device's fitness
    gen.update(fpos, fneg)
    w, n_ranked = orc.centered_ranker(fp.reshape(-1, 1), fn.reshape(-1, 1))
    assert np.array_equal(gen.weights.cpu().numpy(), np.asarray(w).reshape(-1))
    flat = theta.copy()
    orc.approx_grad(flat, orc.SGDOracle(P, 0.01), np.asarray(w).reshape(-1), idx, n_ranked, table, 500, 0.005)
    assert np.abs(gen.theta.cpu().numpy() - flat).max() <= 2e-6
