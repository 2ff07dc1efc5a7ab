"""GPU: binned-action policies (FFBinned, src/nn/nn.py:99-117) on the device -- es_rollout_openloop_binned (the general float32
kernel of rollout_f32.cu, and rollout_tcw.cu under ES_ROLLOUT_TC3) and es_rollout_closedloop_mlp_binned (the cluster kernel of rollout_closedw.cu) against the oracle
(oracle.es_oracle.run_model with FFBinned's head), and es.step with FFBinned against its python loop.

An arg-max turns a rounding difference into a different action only when two bins are within that difference of each other.
So every parity problem is first checked on the float64 truth: the smallest gap between the two largest outputs over every
(evaluation, step, action dimension) must exceed DELTA, far above the float32 forward's error (~1e-6 here).  The kernels and
the oracle then take the same decisions, and what follows from them is exact where the kernel sums as the oracle does:
  * open loop, one CTA per evaluation (>= half the SM count of evaluations): rewards are float32 dots of identical actions,
    summed in float64 in step order, and positions float32 sums in step order -- fitness and positions bit for bit;
  * open loop, time split (fewer evaluations): the per-tile partial sums are added in tile order, so fitness may differ from
    the step-order sum by float64 reassociation (<= 1e-12 of the reward mass) and positions by T half-ulps of their magnitude;
  * open loop, ES_ROLLOUT_TC3 (float16 hi + lo operands, three MMAs per product: outputs within ~1e-6 of float64): the same
    decisions and the same float32 per-step rewards, summed in float64 over rows, warps and tiles -- fitness within 1e-12 of the
    reward mass; positions are float64 sums of the actions scaled once, within T ulps of the oracle's float32 running sums;
  * closed loop: the observations follow the kernel's fast tanh (absolute error ~1e-7), which moves no decision, so fitness and
    positions are compared with test_gpu_closed_wide.py's tolerances and the ObStat sums with 1e-4 of their magnitude.
Problems are searched over a few seeds for one that meets the margin; the test asserts that one was found."""
import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu

SIGMA = 0.02
DELTA = 2e-5
LOW = np.array([-0.3, -1.0, 0.1, -2.0, 0.25, -0.05, -1.0, 0.0], dtype=np.float32)
HIGH = np.array([2.7, 1.0, 0.35, -0.5, 3.0, 0.45, 1.0, 0.6], dtype=np.float32)


def _head(adim, bins):
    from es_pytorch_b200.nn.nn import BinnedHead
    return BinnedHead(bins, LOW[:adim].copy(), HIGH[:adim].copy())


def _binned(head):
    """The oracle's description of a binned head."""
    return head.bins, head.low, head.high


def raw_outputs_f64(layers, x: np.ndarray) -> np.ndarray:
    """The float64 truth of the tanh stack's outputs ([..., adim * bins]) for float32 inputs ``x``."""
    h = np.asarray(x, dtype=np.float64)
    for w, b in layers:
        h = np.tanh(h @ np.asarray(w, np.float64).T + np.asarray(b, np.float64))
    return h


def top_two_gap(out: np.ndarray, bins: int) -> float:
    """The smallest gap between the largest and the second largest output of any action dimension's bins in ``out``
    ([..., adim * bins]): the margin by which every arg-max decision is taken."""
    o = np.sort(np.asarray(out).reshape(-1, int(bins)), axis=1)
    return float((o[:, -1] - o[:, -2]).min())


def _layers(theta, table, idx, P, dims, sign, sigma=SIGMA):
    return orc.unflatten(orc.pheno_params(theta, sigma, sign * orc.table_get(table, int(idx), P)), dims)


def _open_problem(obs, hidden, adim, bins, T, n, mean, std, clip, seeds=range(40), scale=0.05):
    """The first seed whose every decision has a float64 margin > DELTA: (dims, P, table, theta, idx, spec, margin)."""
    spec = orc.SyntheticEnvSpec(obs, adim, T)
    dims = orc.layer_dims(obs, hidden, adim * bins)
    P = orc.n_params(dims)
    xs = orc.normalise_obs(spec.obs_stream[:T], mean, std, clip)
    for seed in seeds:
        rs = np.random.RandomState(seed)
        table = rs.randn(P + 20_000).astype(np.float32)
        theta = (rs.randn(P) * scale).astype(np.float32)
        idx = rs.randint(0, 20_000, size=n).astype(np.int64)
        margin = min(top_two_gap(raw_outputs_f64(_layers(theta, table, i, P, dims, s), xs), bins)
                     for i in idx for s in (1.0, -1.0))
        if margin > DELTA:
            return dims, P, table, theta, idx, spec, margin
    raise AssertionError('no seed gives a problem whose decisions all have a float64 margin > DELTA')


def _open_oracle(dims, P, table, theta, idx, spec, head, mean, std, clip, T, sigma=SIGMA):
    fit, pos = np.zeros((2, len(idx))), np.zeros((2, len(idx), 3), dtype=np.float32)
    for k, i in enumerate(idx):
        for s, sign in enumerate((1.0, -1.0)):
            rews, behv, _, _ = orc.run_model(spec, _layers(theta, table, i, P, dims, sign, sigma), mean, std, clip, T,
                                             batched=True, binned=_binned(head))
            fit[s, k] = sum(rews)
            pos[s, k] = np.array(behv[-3:], dtype=np.float32)
    return fit, pos


def _open_device(eng, sizes, table, idx, theta, spec, head, mean, std, clip, T, sigma=SIGMA, mode=None):
    from es_pytorch_b200 import _lib
    n = len(idx)
    obsn = eng.normalise_obs(eng.to_device(spec.obs_stream[:T]), eng.to_device(np.asarray(mean, np.float64)),
                             eng.to_device(np.asarray(std, np.float64)), clip)
    fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
    eng.rollout(eng.to_device(table), eng.to_device(np.asarray(idx, np.int64)), eng.to_device(theta), sigma, sizes, obsn,
                eng.to_device(spec.rew_vec[:T]), spec.pos_scale, fit[0], fit[1], 1, behv[0].view(-1), behv[1].view(-1),
                _lib.ES_ROLLOUT_F32 if mode is None else mode, head=head)
    eng.sync()
    return fit.cpu().numpy(), behv.cpu().numpy()


def _norm(obs, seed=11):
    rs = np.random.RandomState(seed)
    return rs.randn(obs) * 0.05, 0.5 + rs.rand(obs), 0.8


@pytest.mark.parametrize('hidden,adim,bins,T', [((64, 64), 3, 5, 32), ((64, 64), 6, 11, 8), ((256, 256), 3, 5, 32),
                                                ((256, 256), 3, 11, 32), ((128, 256, 128), 2, 32, 4), ((64, 64), 1, 2, 32)])
def test_open_loop_f32_is_exact_one_cta_per_evaluation(eng, hidden, adim, bins, T):
    """At least half the SM count of evaluations (no time split; 256-wide trunks stage their weights in the global scratch):
    every decision with a float64 margin > DELTA, fitness and positions bit for bit the oracle's.  (Episodes are shorter for the
    heads with more outputs, whose decisions are closer: a problem that meets the margin is then found among the seeds.)"""
    obs = 15
    n = (eng.sm_count + 1) // 2 + 3
    mean, std, clip = _norm(obs)
    head = _head(adim, bins)
    dims, P, table, theta, idx, spec, margin = _open_problem(obs, hidden, adim, bins, T, n, mean, std, clip,
                                                             scale=0.1 if max(hidden) <= 64 else 0.05)
    sizes = [obs, *hidden, adim * bins]
    f, b = _open_device(eng, sizes, table, idx, theta, spec, head, mean, std, clip, T)
    wf, wb = _open_oracle(dims, P, table, theta, idx, spec, head, mean, std, clip, T)
    assert np.array_equal(f, wf), (margin, np.abs(f - wf).max())
    assert np.array_equal(b, wb), (margin, np.abs(b - wb).max())
    # the same evaluations in reverse order: bit-identical
    fr, br = _open_device(eng, sizes, table, idx[::-1].copy(), theta, spec, head, mean, std, clip, T)
    assert np.array_equal(fr[:, ::-1], f) and np.array_equal(br[:, ::-1], b)


@pytest.mark.parametrize('hidden,n_pairs,T', [((64, 64), 1, 200), ((256, 256), 2, 131), ((64, 64), 5, 1)])
def test_open_loop_f32_time_split(eng, hidden, n_pairs, T):
    """Fewer evaluations than SMs: the episode's time tiles are split over the idle SMs.  Same decisions; fitness within float64
    reassociation of the oracle's step-order sum, positions within T half-ulps."""
    obs, adim, bins = 15, 3, 5
    mean, std, clip = _norm(obs)
    head = _head(adim, bins)
    dims, P, table, theta, idx, spec, margin = _open_problem(obs, hidden, adim, bins, T, n_pairs, mean, std, clip)
    f, b = _open_device(eng, [obs, *hidden, adim * bins], table, idx, theta, spec, head, mean, std, clip, T)
    wf, wb = _open_oracle(dims, P, table, theta, idx, spec, head, mean, std, clip, T)
    mass = max(1.0, float(np.abs(spec.rew_vec[:T]).sum() * np.abs(np.concatenate([LOW, HIGH])).max()))
    assert np.abs(f - wf).max() <= 1e-12 * mass, (margin, np.abs(f - wf).max())
    assert np.abs(b - wb).max() <= T * 0.5 * np.spacing(np.float32(max(1.0, np.abs(wb).max()))), np.abs(b - wb).max()


@pytest.mark.parametrize('obs,hidden,adim,bins,T', [(15, (64, 64), 3, 5, 32), (15, (256, 256), 3, 11, 32),
                                                    (17, (256, 256, 256), 6, 5, 16), (28, (128, 256, 256, 128), 8, 11, 8),
                                                    (256, (64, 128), 4, 64, 8), (15, (256, 256), 1, 2, 300)])
def test_open_loop_tc3_takes_the_same_decisions(eng, obs, hidden, adim, bins, T):
    """ES_ROLLOUT_TC3 (rollout_tcw.cu, obs-64-64-X included): same margin-checked problems, same decisions; fitness within
    1e-12 of the reward mass of the float64-exact step-order sum of the same float32 rewards, positions within T ulps."""
    from es_pytorch_b200 import _lib
    n = 20
    mean, std, clip = _norm(obs)
    head = _head(adim, bins)
    dims, P, table, theta, idx, spec, margin = _open_problem(obs, hidden, adim, bins, T, n, mean, std, clip,
                                                             scale=0.1 if max(hidden) <= 64 else 0.05)
    sizes = [obs, *hidden, adim * bins]
    f, b = _open_device(eng, sizes, table, idx, theta, spec, head, mean, std, clip, T, mode=_lib.ES_ROLLOUT_TC3)
    wf, wb = _open_oracle(dims, P, table, theta, idx, spec, head, mean, std, clip, T)
    mass = max(1.0, float(np.abs(spec.rew_vec[:T]).sum() * np.abs(np.concatenate([LOW, HIGH])).max()))
    assert np.abs(f - wf).max() <= 1e-12 * mass, (margin, np.abs(f - wf).max())
    assert np.abs(b - wb).max() <= T * np.spacing(np.float32(max(1.0, np.abs(wb).max()))), np.abs(b - wb).max()
    fr, br = _open_device(eng, sizes, table, idx[::-1].copy(), theta, spec, head, mean, std, clip, T, mode=_lib.ES_ROLLOUT_TC3)
    assert np.array_equal(fr[:, ::-1], f) and np.array_equal(br[:, ::-1], b)


def _tie_theta(rs, dims, P, bins, winners=None):
    """Random trunk, last layer weights 0 and equal biases (an exact tie in every dimension), or a strictly larger bias on bin
    winners[j] of dimension j."""
    theta = (rs.randn(P) * 0.1).astype(np.float32)
    layers = orc.unflatten(theta, dims)          # views into theta
    w, b = layers[-1]
    w[...] = 0.0
    b[...] = np.float32(0.2)
    if winners is not None:
        for j, k in enumerate(winners):
            b[j * bins + k] = np.float32(0.3)
    return theta


@pytest.mark.parametrize('hidden,n_pairs,tc3', [((64, 64), 70, False), ((64, 64), 1, False), ((256, 256), 70, False),
                                                ((64, 64), 4, True), ((256, 256), 4, True)])
def test_exact_ties_take_the_first_bin_open_loop(eng, hidden, n_pairs, tc3):
    """Last layer 0 with equal biases: bin 0 (action = low) on every step; a strictly larger bias on bin k: bin k.  sigma = 0.
    On the float32 kernel (one CTA per evaluation, and time split) and on ES_ROLLOUT_TC3."""
    from es_pytorch_b200 import _lib
    obs, adim, bins, T = 15, 3, 5, 40
    dims = orc.layer_dims(obs, hidden, adim * bins)
    P = orc.n_params(dims)
    rs = np.random.RandomState(5)
    table = rs.randn(P + 1000).astype(np.float32)
    spec = orc.SyntheticEnvSpec(obs, adim, T)
    head = _head(adim, bins)
    z, o = np.zeros(obs), np.ones(obs)
    idx = np.zeros(n_pairs, dtype=np.int64)
    for winners in (None, [4, 0, 2]):
        theta = _tie_theta(rs, dims, P, bins, winners)
        f, b = _open_device(eng, [obs, *hidden, adim * bins], table, idx, theta, spec, head, z, o, 5.0, T, sigma=0.0,
                            mode=_lib.ES_ROLLOUT_TC3 if tc3 else _lib.ES_ROLLOUT_F32)
        a = head.low if winners is None else orc.binned_action(np.eye(bins, dtype=np.float32)[winners].reshape(-1), bins,
                                                                    head.low, head.high)
        rews, behv, _, _ = orc.run_model(spec, orc.unflatten(theta, dims), z, o, 5.0, T, binned=_binned(head))
        acc = [np.float32(0)] * T
        for t in range(T):
            for j in range(adim):
                acc[t] = np.float32(acc[t] + np.float32(a[j] * spec.rew_vec[t, j]))
        assert np.array_equal(np.array(rews, np.float32), np.array(acc, np.float32))      # the oracle takes the same bins
        exact = not tc3 and 2 * n_pairs >= eng.sm_count
        assert np.all(f == sum(rews)) if exact else np.abs(f - sum(rews)).max() <= 1e-12 * max(1, T)
        assert np.abs(b - np.array(behv[-3:], np.float32)).max() <= T * np.spacing(np.float32(max(1.0, np.abs(behv[-3:]).max())))


# ------------------------------------------------------------------------------------------------------------------ closed loop
def _closed_problem(obs, hidden, adim, bins, T, n, mean, std, clip, band=8, seeds=range(40), scale=0.03, delta=1e-4):
    spec = orc.ClosedLoopEnvSpec(obs, adim, T, band=band)
    dims = orc.layer_dims(obs, hidden, adim * bins)
    P = orc.n_params(dims)
    head = _head(adim, bins)
    for seed in seeds:
        rs = np.random.RandomState(seed)
        table = rs.randn(P + 20_000).astype(np.float32)
        theta = (rs.randn(P) * scale).astype(np.float32)
        idx = rs.randint(0, 20_000, size=n).astype(np.int64)
        margin = np.inf
        for i in idx:
            for s in (1.0, -1.0):
                layers = _layers(theta, table, i, P, dims, s)
                _, _, obs_after, _ = orc.run_model(spec, layers, mean, std, clip, T, binned=_binned(head))
                # the normalised observations the network saw: obs_0, then every post-step observation but the last
                xs = orc.normalise_obs(np.concatenate([spec.obs_stream[:1], obs_after[:-1]]), mean, std, clip)
                margin = min(margin, top_two_gap(raw_outputs_f64(layers, xs), bins))
        if margin > delta:
            return dims, P, table, theta, idx, spec, margin
    raise AssertionError('no seed gives a closed-loop problem whose decisions all have a float64 margin > delta')


def _assert_contractive(spec, layers, mean, std, clip, head, steps=150):
    s = orc.ClosedLoopEnvSpec(spec.obs_dim, spec.act_dim, steps, band=spec.band)
    _, _, a, _ = orc.run_model(s, layers, mean, std, clip, steps, binned=_binned(head))
    s.obs_stream = s.obs_stream.copy()
    s.obs_stream[0] += np.float32(0.3)
    _, _, b, _ = orc.run_model(s, layers, mean, std, clip, steps, binned=_binned(head))
    assert np.abs(a[-1] - b[-1]).max() < 1e-6, 'the loop is not contractive at this shape: the comparison would mean nothing'


def _closed_device(eng, sizes, table, idx, theta, spec, head, mean, std, clip, coins=None, sigma=SIGMA):
    n, obs = len(idx), sizes[0]
    fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
    osum, osq = (torch.zeros(obs, dtype=torch.float64, device=eng.device) for _ in range(2))
    ocnt = torch.zeros(2, dtype=torch.float64, device=eng.device)
    eng.rollout_closed_mlp(eng.to_device(table), eng.to_device(np.asarray(idx, np.int64)), eng.to_device(theta), sigma, sizes,
                           eng.to_device(np.asarray(mean, np.float64)), eng.to_device(np.asarray(std, np.float64)), clip,
                           eng.to_device(spec.obs_stream[0].copy()), eng.to_device(np.ascontiguousarray(spec.env_a.T)),
                           eng.to_device(np.ascontiguousarray(spec.env_b.T)), eng.to_device(spec.rew_vec), spec.pos_scale,
                           fit[0], fit[1], 1, behv[0].view(-1), behv[1].view(-1),
                           coin_words=None if coins is None else eng.to_device(coins.view(np.int32)), save_obs_chance=0.5,
                           ob_sum=osum, ob_sumsq=osq, ob_count=ocnt, head=head)
    eng.sync()
    return fit.cpu().numpy(), behv.cpu().numpy(), osum.cpu().numpy(), osq.cpu().numpy(), ocnt.cpu().numpy()


def _coins(n, saved):
    """Coin words [n][+,-][2]: evaluation e saves (random_sample < 0.5) iff saved[e]."""
    coins = np.full((n, 4), 0xFFFFFFFF, dtype=np.uint32)
    for e, s in enumerate(saved):
        if s:
            coins[e // 2, 2 * (e % 2):2 * (e % 2) + 2] = 0
    return coins


@pytest.mark.parametrize('obs,hidden,adim,bins', [(15, (64, 64), 3, 5), (15, (256, 256), 3, 11), (17, (256, 256, 256), 6, 5),
                                                  (28, (128, 256, 256, 128), 8, 11), (8, (16, 16), 2, 2)])
def test_closed_loop_cluster_against_the_oracle(eng, obs, hidden, adim, bins):
    """es_rollout_closedloop_mlp_binned against the oracle's per-step loop, with coins (some evaluations save their
    observations); the plan's cluster size (one CTA for the small shape); bit-identical when the pairs are reversed."""
    T, n = 48, 4
    mean, std, clip = _norm(obs)
    head = _head(adim, bins)
    dims, P, table, theta, idx, spec, margin = _closed_problem(obs, hidden, adim, bins, T, n, mean, std, clip)
    _assert_contractive(spec, orc.unflatten(theta, dims), mean, std, clip, head)
    sizes = [obs, *hidden, adim * bins]
    C, clusters, smem = eng.closed_mlp_plan(sizes, spec.band, head)
    assert C >= 1 and clusters >= 1 and smem > 0
    if hidden == (16, 16):
        assert C == 1
    saved = [e % 3 == 0 for e in range(2 * n)]
    f, b, osum, osq, ocnt = _closed_device(eng, sizes, table, idx, theta, spec, head, mean, std, clip, coins=_coins(n, saved))
    stat = orc.ObStatOracle((obs,), 0)
    for k, i in enumerate(idx):
        for s, sign in enumerate((1.0, -1.0)):
            rews, behv, obsv, _ = orc.run_model(spec, _layers(theta, table, i, P, dims, sign), mean, std, clip, T,
                                                binned=_binned(head))
            assert abs(f[s, k] - sum(rews)) <= 2e-5 * max(1.0, np.abs(rews).sum()), (margin, k, s)
            assert np.abs(b[s, k] - np.array(behv[-3:], np.float32)).max() <= 1e-5
            if saved[2 * k + s]:
                stat.inc(*orc.ob_sum_sq_cnt(obsv))
    assert ocnt[0] == stat.count and ocnt[1] == sum(saved)
    assert np.abs(osum - stat.sum).max() <= 1e-4 * max(1.0, np.abs(stat.sum).max())
    assert np.abs(osq - stat.sumsq).max() <= 1e-4 * max(1.0, np.abs(stat.sumsq).max())
    fr, br, _, _, _ = _closed_device(eng, sizes, table, idx[::-1].copy(), theta, spec, head, mean, std, clip)
    assert np.array_equal(fr[:, ::-1], f) and np.array_equal(br[:, ::-1], b)


def test_exact_ties_take_the_first_bin_closed_loop(eng):
    obs, hidden, adim, bins, T = 15, (64, 64), 3, 5, 40
    dims = orc.layer_dims(obs, hidden, adim * bins)
    P = orc.n_params(dims)
    rs = np.random.RandomState(6)
    table = rs.randn(P + 1000).astype(np.float32)
    spec = orc.ClosedLoopEnvSpec(obs, adim, T)
    head = _head(adim, bins)
    z, o = np.zeros(obs), np.ones(obs)
    for winners in (None, [1, 4, 3]):
        theta = _tie_theta(rs, dims, P, bins, winners)
        f, b, _, _, _ = _closed_device(eng, [obs, *hidden, adim * bins], table, np.zeros(2, np.int64), theta, spec, head, z, o,
                                       5.0, sigma=0.0)
        rews, behv, _, _ = orc.run_model(spec, orc.unflatten(theta, dims), z, o, 5.0, T, binned=_binned(head))
        assert np.all(f == sum(rews)) and np.all(b == np.array(behv[-3:], np.float32))


# ------------------------------------------------------------------------------------------------------------------ refusals
def test_refusals(eng):
    from es_pytorch_b200 import _lib
    from es_pytorch_b200.nn.nn import BinnedHead
    obs, hidden, adim, bins, T = 15, (64, 64), 3, 5, 8
    spec = orc.SyntheticEnvSpec(obs, adim, T)
    cspec = orc.ClosedLoopEnvSpec(obs, adim, T)
    z, o = np.zeros(obs), np.ones(obs)

    def run(sizes, head, mode=_lib.ES_ROLLOUT_F32, o_=obs, sp=spec):
        P = orc.n_params(orc.layer_dims(sizes[0], sizes[1:-1], sizes[-1]))
        table = np.zeros(P + 10, np.float32)
        return _open_device(eng, sizes, table, [0], np.zeros(P, np.float32), sp, head, np.zeros(o_), np.ones(o_), 5.0, T,
                            mode=mode)

    def raises(fn, *words):
        with pytest.raises(_lib.EsLibraryError) as exc:
            fn()
        for w in words:
            assert w in str(exc.value), str(exc.value)

    sizes = [obs, *hidden, adim * bins]
    raises(lambda: run(sizes, _head(adim, bins), _lib.ES_ROLLOUT_TC), 'ES_ROLLOUT_TC refuses', 'parity', 'code -3')
    raises(lambda: run([257, 64, 64, adim * bins], _head(adim, bins), _lib.ES_ROLLOUT_TC3, 257,
                       orc.SyntheticEnvSpec(257, adim, T)), 'ES_ROLLOUT_TC3', 'got obs 257', 'code -3')
    raises(lambda: run([obs, 96, 64, adim * bins], _head(adim, bins), _lib.ES_ROLLOUT_TC3), 'got hidden layer 1 of width 96',
           'code -3')
    raises(lambda: run([obs, 64, 64, 64, 64, 64, adim * bins], _head(adim, bins), _lib.ES_ROLLOUT_TC3), 'got 5 hidden layers',
           'code -3')
    raises(lambda: run([obs, 64, 64, 3 * 86], _head(3, 86), _lib.ES_ROLLOUT_TC3), '256', 'code -3')
    raises(lambda: run([obs, 64, 64, 3], BinnedHead(1, LOW[:3].copy(), HIGH[:3].copy())), 'bins must be >= 2', 'code -1')
    raises(lambda: run([obs, 64, 64, 3 * 86], _head(3, 86)), '256', 'code -3')
    P = orc.n_params(orc.layer_dims(obs, hidden, 3 * 86))
    raises(lambda: _closed_device(eng, [obs, 64, 64, 3 * 86], np.zeros(P + 10, np.float32), [0], np.zeros(P, np.float32), cspec,
                                  _head(3, 86), z, o, 5.0), '256', 'code -3')
    raises(lambda: eng.closed_mlp_plan([obs, 64, 64, 3], 8, BinnedHead(1, LOW[:3].copy(), HIGH[:3].copy())), 'bins', 'code -1')
    raises(lambda: eng.closed_mlp_plan([obs, 64, 64, 3 * 86], 8, _head(3, 86)), '256', 'code -3')
    # the tanh paths are untouched by a head of 'tanh'
    P = orc.n_params(orc.layer_dims(obs, hidden, adim))
    f, _ = _open_device(eng, [obs, *hidden, adim], np.zeros(P + 10, np.float32), [0], np.zeros(P, np.float32), spec, 'tanh', z, o,
                        5.0, T)
    assert np.all(f == 0.0)


# ------------------------------------------------------------------------------------------------------------------ es.step
class _PlainEnv:
    """The synthetic env without its open-loop marker: run_model steps it in the python loop through the module's forward."""

    def __init__(self, env):
        self._env = env

    def __getattr__(self, name):
        if name == 'is_synthetic_openloop':
            raise AttributeError(name)
        return getattr(self._env, name)


def _steps(closed, archive=None, gens=2):
    """es.step with FFBinned through a BatchedRollout (one fused device generation) and through an opaque fit_fn that runs
    run_model's python loop (FFBinned.forward at every step), from the same theta, table and streams."""
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    from es_pytorch_b200.gym.training_result import NSRResult, RewardResult
    from es_pytorch_b200.nn.nn import FFBinned
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker, MultiObjectiveRanker
    from es_pytorch_b200.utils.reporters import Reporter

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    obs, act, T, n, bins, chance = 15, 3, 24, 8, 5, 0.3
    env = (ClosedLoopEnv if closed else SyntheticEnv)(obs, act, T)
    env.action_space.low = LOW[:act].copy()
    env.action_space.high = HIGH[:act].copy()
    nets = [FFBinned([64, 64], torch.nn.Tanh(), env, bins, 5) for _ in range(2)]
    P = len(Policy.get_flat(nets[0]))
    rs = np.random.RandomState(21)
    table = rs.randn(P + 50_000).astype(np.float32)
    theta = (rs.randn(P) * 0.1).astype(np.float32)
    policies = []
    for net in nets:
        p = Policy(net, SIGMA, Adam(P, 0.01))
        p.flat_params[...] = theta
        p.set_nn_params(p.flat_params)
        policies.append(p)
    nts = [NoiseTable(P, table.copy()) for _ in range(2)]
    streams = [np.random.RandomState(77), np.random.RandomState(77)]
    rankers = [MultiObjectiveRanker(CenteredRanker(), 0.5) if archive is not None else CenteredRanker() for _ in range(2)]
    cfg = Cfg(general=Cfg(policies_per_gen=2 * n, batch_size=500), policy=Cfg(l2coeff=0.005))
    fused = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=chance, archive=archive, nov_k=5)
    step_env = env if closed else _PlainEnv(env)
    zeros = np.array([np.zeros(obs)])

    def opaque(model, use_ac_noise=True):             # the scripts' fit_fn (simple_example.py / nsra.py), python loop
        save = streams[1].random() < chance
        rews, behv, obsv, steps = run_model(model, step_env, T, None)
        o = obsv if save else zeros
        if archive is None:
            return RewardResult(rews, behv, o, steps)
        return NSRResult(rews, behv[-3:], o, steps, archive, 5)

    assert es._can_fuse_step(dist.world(), policies[0], fused, rankers[0])
    assert not es._can_fuse_step(dist.world(), policies[1], opaque, rankers[1])
    out = []
    for g in range(gens):
        res = []
        for p, nt, fit_fn, st, rk in zip(policies, nts, (fused, opaque), streams, rankers):
            tr, gen_obstat = es.step(cfg, dist.world(), p, nt, env, fit_fn, st, rk, Reporter())
            p.update_obstat(gen_obstat)
            res.append((tr, gen_obstat, np.asarray(rk.noise_inds).copy(), np.asarray(rk.ranked_fits).copy(),
                        np.concatenate((np.asarray(rk.fits_pos), np.asarray(rk.fits_neg))), p.flat_params.copy()))
        out.append(res)
        assert np.array_equal(streams[0].get_state()[1], streams[1].get_state()[1])
        assert streams[0].get_state()[2] == streams[1].get_state()[2]
    return out


def _assert_same_steps(out, fit_tol):
    for g, ((tr_a, st_a, ia, wa, fa, th_a), (tr_b, st_b, ib, wb, fb, th_b)) in enumerate(out):
        assert np.array_equal(ia, ib), g
        assert np.abs(fa - fb).max() <= fit_tol, (g, np.abs(fa - fb).max())
        assert np.array_equal(wa, wb), g
        assert np.abs(th_a - th_b).max() <= 3e-6, (g, np.abs(th_a - th_b).max())
        assert st_a.count == st_b.count and st_a.count > 0
        assert np.abs(st_a.sum - st_b.sum).max() <= 1e-4 * max(1.0, np.abs(st_b.sum).max())
        assert abs(tr_a.result[0] - tr_b.result[0]) <= max(fit_tol, 1e-9), (g, tr_a.result, tr_b.result)


def test_es_step_fused_open_loop_matches_the_python_loop(eng):
    """Open loop: same decisions, so the fused fitness IS the python loop's (float32 rewards summed in step order)."""
    _assert_same_steps(_steps(closed=False), 0.0)


def test_es_step_fused_closed_loop_matches_the_python_loop(eng):
    _assert_same_steps(_steps(closed=True), 2e-5 * 24 * 3)


def test_es_step_fused_nsra_generation_matches_the_python_loop(eng):
    """NSRA: the novelty of the final position, computed on the device from the binned actions' positions."""
    archive = np.random.RandomState(17).randn(12, 2) * 0.05
    _assert_same_steps(_steps(closed=False, archive=archive, gens=1), 1e-12)


def test_batched_rollout_call_runs_a_binned_policy_as_one_episode_launch(eng):
    """The per-call fit_fn (es.step's noiseless evaluation, the call-by-call route): the closed loop as one launch of the cluster
    kernel, the open loop as the observation normalisation plus one rollout; both against run_model's python loop."""
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    from es_pytorch_b200.nn.nn import FFBinned
    T = 40
    for closed in (False, True):
        env = (ClosedLoopEnv if closed else SyntheticEnv)(15, 3, T)
        env.action_space.low = LOW[:3].copy()
        env.action_space.high = HIGH[:3].copy()
        torch.manual_seed(4)
        net = FFBinned([64, 64], torch.nn.Tanh(), env, 5)
        fit_fn = BatchedRollout(env, T, coins_per_eval=0)
        l0 = eng.launches
        got = fit_fn(net, False).result[0]
        assert eng.launches - l0 == (1 if closed else 2)
        rews, _, _, _ = run_model(net, env if closed else _PlainEnv(env), T, None)
        if closed:
            assert abs(got - sum(rews)) <= 2e-5 * max(1.0, np.abs(rews).sum())
        else:
            assert got == sum(rews)
