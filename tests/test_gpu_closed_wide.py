"""GPU parity of the closed-loop synthetic env at the shipped configs' wide policies (es_rollout_closedloop_mlp: one thread-block
cluster per evaluation, rollout_closedw.cu), against the oracle's literal per-step loop (oracle.es_oracle.run_model).

Tolerances are test_gpu_closed.py's: fitness |f - oracle| <= 2e-5 max(1, sum |r|), positions 1e-5.  They only mean something
where the loop forgets rounding differences, so every shape is first checked on the oracle to be contractive: a start
observation moved by 0.3 is forgotten within the episode (theta scale 0.03, sigma 0.02, std O(1) and an active clip).

The long episodes (T = 1 000 and 10 000) widen two bounds by the rounding of float32 running sums, which both sides perform:
the position adds T float32 terms and the ObStat column sums T per saved evaluation, each addition rounding by up to half an
ulp of the sum.  Once the two sides' terms differ in their last bits those roundings differ too, so the sums may part by up to
T ulps of their magnitude (an analytic bound: 1.2e-4 for simple_conf's positions, where 1.1e-5 was seen on an H100)."""
import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu

SIGMA = 0.02


def _problem(obs, hidden, act, T, seed=3, scale=0.03, band=8, table_extra=50_000):
    dims = orc.layer_dims(obs, hidden, act)
    P = orc.n_params(dims)
    rs = np.random.RandomState(seed)
    table = rs.randn(P + table_extra).astype(np.float32)
    theta = (rs.randn(P) * scale).astype(np.float32)
    return dims, P, table, theta, orc.ClosedLoopEnvSpec(obs, act, T, band=band)


def _norm(obs, seed=11):
    """A non-trivial normalisation: mean != 0, std O(1) and a clip that is active (the observations reach +-1)."""
    rs = np.random.RandomState(seed)
    return rs.randn(obs) * 0.05, 0.5 + rs.rand(obs), 0.4


def _dev_env(eng, spec):
    return (eng.to_device(spec.obs_stream[0].copy()), eng.to_device(np.ascontiguousarray(spec.env_a.T)),
            eng.to_device(np.ascontiguousarray(spec.env_b.T)))


def _layers(theta, table, idx, P, dims, sign, sigma=SIGMA):
    return orc.unflatten(orc.pheno_params(theta, sigma, sign * orc.table_get(table, int(idx), P)), dims)


def _assert_contractive(spec, layers, mean, std, clip, steps=150):
    s = orc.ClosedLoopEnvSpec(spec.obs_dim, spec.act_dim, steps, band=spec.band)
    _, _, a, _ = orc.run_model(s, layers, mean, std, clip, steps)
    s.obs_stream = s.obs_stream.copy()
    s.obs_stream[0] += np.float32(0.3)
    _, _, b, _ = orc.run_model(s, layers, mean, std, clip, steps)
    assert np.abs(a[-1] - b[-1]).max() < 1e-6, 'the loop is not contractive at this shape: the comparison would mean nothing'


class _Run:
    """One es_rollout_closedloop_mlp call with every output: fit [2][n * stride], behv [2][n][3], ObStat sums and counts."""

    def __init__(self, eng, sizes, table, idx, theta, spec, mean, std, clip, sigma=SIGMA, coins=None, fit_stride=1,
                 stats=True, behv=True):
        n, obs = len(idx), sizes[0]
        self.fit = torch.zeros(2, max(1, n * fit_stride), dtype=torch.float64, device=eng.device)
        self.behv = torch.zeros(2, max(1, n), 3, dtype=torch.float32, device=eng.device) if behv else None
        self.osum, self.osq = (torch.zeros(obs, dtype=torch.float64, device=eng.device) for _ in range(2))
        self.ocnt = torch.zeros(2, dtype=torch.float64, device=eng.device)
        obs0, env_a, env_b = _dev_env(eng, spec)
        eng.rollout_closed_mlp(eng.to_device(table), eng.to_device(np.asarray(idx, np.int64)), eng.to_device(theta), sigma, sizes,
                               eng.to_device(mean), eng.to_device(std), clip, obs0, env_a, env_b, eng.to_device(spec.rew_vec),
                               spec.pos_scale, self.fit[0], self.fit[1], fit_stride,
                               None if not behv else self.behv[0].view(-1), None if not behv else self.behv[1].view(-1),
                               coin_words=None if coins is None else eng.to_device(coins.view(np.int32)), save_obs_chance=0.5,
                               ob_sum=self.osum if stats else None, ob_sumsq=self.osq if stats else None,
                               ob_count=self.ocnt if stats else None)
        eng.sync()
        self.f = self.fit.cpu().numpy()[:, ::fit_stride][:, :n]
        self.b = None if not behv else self.behv.cpu().numpy()[:, :n]


def _coins(n, saved):
    coins = np.full((n, 4), 0xFFFFFFFF, dtype=np.uint32)
    for k, sgn in saved:
        coins[k, 2 * sgn:2 * sgn + 2] = 0                                           # u = 0 < chance
    return coins


def _check_against_oracle(run, table, theta, idx, P, dims, spec, mean, std, clip, T, pairs, saved=(), sigma=SIGMA):
    ref_sum, ref_sq = np.zeros(spec.obs_dim), np.zeros(spec.obs_dim)
    for k in pairs:
        for sgn, sign in enumerate((1.0, -1.0)):
            rews, bh, obs, _ = orc.run_model(spec, _layers(theta, table, idx[k], P, dims, sign, sigma), mean, std, clip, T)
            want = orc.reward_result(rews)[0]
            assert abs(run.f[sgn, k] - want) <= 2e-5 * max(1.0, np.abs(rews).sum()), (k, sgn, run.f[sgn, k], want)
            if run.b is not None:
                pos_tol = max(1e-5, T * float(np.spacing(np.float32(np.abs(bh[-3:]).max()))))
                assert np.abs(run.b[sgn, k] - np.array(bh[-3:])).max() <= pos_tol, (k, sgn)
            if (k, sgn) in saved:
                ref_sum += obs.sum(axis=0).astype(np.float64)
                ref_sq += np.square(obs).sum(axis=0).astype(np.float64)
    return ref_sum, ref_sq


# the shipped configs' policies (simple_conf / nsra, obj, the 26-wide variant, ns, flagrun) and a Humanoid-shaped wide one
SHIPPED = [
    ('simple_conf_nsra', 15, (256, 256), 3, 1000, 3, 2),
    ('obj', 17, (256, 256, 256), 6, 300, 3, 1),
    ('obj26', 26, (256, 256, 256), 6, 300, 3, 1),
    ('ns', 28, (256, 256, 256), 8, 10_000, 2, 1),
    ('flagrun', 28, (128, 256, 256, 128), 8, 300, 3, 1),
    ('humanoid_wide', 376, (256, 256), 17, 200, 3, 1),
]


@pytest.mark.parametrize('name,obs,hidden,act,T,n_pairs,fit_stride', SHIPPED, ids=[c[0] for c in SHIPPED])
def test_closed_wide_shipped_shapes_match_the_oracle(eng, name, obs, hidden, act, T, n_pairs, fit_stride):
    """Fitness, final position and the ObStat increments of the saved rollouts; simple_conf with nsra's layout (fit_stride 2)."""
    dims, P, table, theta, spec = _problem(obs, hidden, act, T)
    mean, std, clip = _norm(obs)
    idx = np.random.RandomState(7).randint(0, len(table) - P, size=n_pairs).astype(np.int64)
    _assert_contractive(spec, _layers(theta, table, idx[0], P, dims, 1.0), mean, std, clip)
    sizes = [obs, *hidden, act]
    assert eng.closed_mlp_plan(sizes, spec.band)[0] >= 1                          # the cluster kernel, not rollout_closed.cu
    saved = [(k, sgn) for k in range(n_pairs) for sgn in range(2) if (k + sgn) % 2 == 0]
    run = _Run(eng, sizes, table, idx, theta, spec, mean, std, clip, coins=_coins(n_pairs, saved), fit_stride=fit_stride)
    if fit_stride > 1:
        assert not run.fit.cpu().numpy()[:, 1::fit_stride].any()                   # the other objective's column is untouched
    ref_sum, ref_sq = _check_against_oracle(run, table, theta, idx, P, dims, spec, mean, std, clip, T, range(n_pairs), saved)
    assert run.ocnt.cpu().numpy().tolist() == [float(len(saved) * T), float(len(saved))]
    for got, ref in ((run.osum.cpu().numpy(), ref_sum), (run.osq.cpu().numpy(), ref_sq)):
        per_eval = np.float32(np.abs(ref).max() / max(1, len(saved)))
        tol = max(1e-4 * max(1.0, np.abs(ref).max()), len(saved) * T * float(np.spacing(per_eval)))
        assert np.abs(got - ref).max() <= tol


EDGES = [  # (obs, hidden, act, band, T)
    (20, (1, 65), 5, 8, 40),                # width 1, and 65 (just past rollout_closed.cu's 64)
    (20, (255, 256), 5, 8, 40),
    (20, (65, 1, 255), 3, 8, 40),           # mixed widths, three hidden layers
    (24, (96, 200, 33, 130), 7, 4, 40),     # four hidden layers, ragged
    (20, (96, 80), 1, 8, 40),               # act 1
    (20, (130, 70), 64, 8, 40),             # act 64
    (8, (100, 100), 4, 8, 40),              # obs == band
    (384, (128, 128), 8, 16, 30),           # obs 384, band 16
    (15, (256, 256), 3, 8, 1),              # T = 1
    (15, (256, 256), 3, 8, 2),              # T = 2
]


@pytest.mark.parametrize('obs,hidden,act,band,T', EDGES)
def test_closed_wide_edges_match_the_oracle(eng, obs, hidden, act, band, T):
    dims, P, table, theta, spec = _problem(obs, hidden, act, T, band=band)
    mean, std, clip = _norm(obs)
    idx = np.random.RandomState(5).randint(0, len(table) - P, size=2).astype(np.int64)
    _assert_contractive(spec, _layers(theta, table, idx[0], P, dims, 1.0), mean, std, clip)
    sizes = [obs, *hidden, act]
    assert eng.closed_mlp_plan(sizes, band)[0] >= 1
    saved = [(0, 1), (1, 0)]
    run = _Run(eng, sizes, table, idx, theta, spec, mean, std, clip, coins=_coins(2, saved))
    ref_sum, _ = _check_against_oracle(run, table, theta, idx, P, dims, spec, mean, std, clip, T, range(2), saved)
    assert run.ocnt.cpu().numpy().tolist() == [float(2 * T), 2.0]
    assert np.abs(run.osum.cpu().numpy() - ref_sum).max() <= 1e-4 * max(1.0, np.abs(ref_sum).max())


def _largest_fitting_width(eng):
    """The family 384-256-256-h-64 (band 16): the largest h whose weights and env matrices fit a cluster of 8 CTAs."""
    from es_pytorch_b200._lib import EsLibraryError

    def fits(h):
        try:
            eng.closed_mlp_plan([384, 256, 256, h, 64], 16)
            return True
        except EsLibraryError:
            return False
    lo, hi = 1, 256
    assert fits(lo) and not fits(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid)
    return lo


def test_closed_wide_largest_shape_in_eight_ctas(eng):
    """The largest shape of a family that fits 8 CTAs runs (and matches the oracle); one unit more is refused, naming bytes."""
    from es_pytorch_b200._lib import EsLibraryError
    h = _largest_fitting_width(eng)
    assert eng.closed_mlp_plan([384, 256, 256, h, 64], 16)[0] == 8
    with pytest.raises(EsLibraryError, match='bytes of shared memory per CTA in a cluster of 8'):
        eng.closed_mlp_plan([384, 256, 256, h + 1, 64], 16)
    T = 12
    dims, P, table, theta, spec = _problem(384, (256, 256, h), 64, T, band=16)
    mean, std, clip = _norm(384)
    idx = np.array([17, 4321], dtype=np.int64)
    _assert_contractive(spec, _layers(theta, table, idx[0], P, dims, 1.0), mean, std, clip)
    run = _Run(eng, [384, 256, 256, h, 64], table, idx, theta, spec, mean, std, clip)
    _check_against_oracle(run, table, theta, idx, P, dims, spec, mean, std, clip, T, range(2))


def test_closed_wide_pair_counts_and_order(eng):
    """1 pair, around the resident clusters (in pairs and in evaluations) and a larger multiple: each run matches the oracle on
    its first and last pair and is bit-identical to the run of the same pairs in reverse order."""
    obs, hidden, act, T = 15, (256, 256), 3, 20
    dims, P, table, theta, spec = _problem(obs, hidden, act, T)
    mean, std, clip = _norm(obs)
    sizes = [obs, *hidden, act]
    C, n_cl, smem = eng.closed_mlp_plan(sizes, spec.band)
    assert C == 2 and 1 <= n_cl <= eng.sm_count // C and smem <= 227 * 1024
    counts = sorted({1, max(1, n_cl // 2 - 1), n_cl // 2 + 1, n_cl - 1, n_cl + 1, 3 * n_cl + 1})
    rs = np.random.RandomState(9)
    for n in counts:
        idx = rs.randint(0, len(table) - P, size=n).astype(np.int64)
        saved = [(k, sgn) for k in range(n) for sgn in range(2) if (k + 2 * sgn) % 3 == 0]
        coins = _coins(n, saved)
        a = _Run(eng, sizes, table, idx, theta, spec, mean, std, clip, coins=coins)
        b = _Run(eng, sizes, table, idx[::-1].copy(), theta, spec, mean, std, clip, coins=coins[::-1].copy())
        assert np.array_equal(a.f, b.f[:, ::-1]) and np.array_equal(a.b, b.b[:, ::-1]), n
        assert a.ocnt.cpu().numpy().tolist() == b.ocnt.cpu().numpy().tolist() == [float(len(saved) * T), float(len(saved))]
        _check_against_oracle(a, table, theta, idx, P, dims, spec, mean, std, clip, T, sorted({0, n - 1}))


def test_closed_wide_sigma_zero_signs_are_identical(eng):
    obs, hidden, act, T = 17, (256, 256, 256), 6, 50
    dims, P, table, theta, spec = _problem(obs, hidden, act, T)
    mean, std, clip = _norm(obs)
    idx = np.random.RandomState(2).randint(0, len(table) - P, size=5).astype(np.int64)
    run = _Run(eng, [obs, *hidden, act], table, idx, theta, spec, mean, std, clip, sigma=0.0)
    assert np.array_equal(run.f[0], run.f[1]) and np.array_equal(run.b[0], run.b[1])
    assert np.all(run.f[0] == run.f[0, 0])
    _check_against_oracle(run, table, theta, idx, P, dims, spec, mean, std, clip, T, [0], sigma=0.0)


def test_closed_wide_dispatch_and_launches(eng):
    """17-64-64-6 through the new entry point runs rollout_closed.cu: bit-identical to es_rollout_closedloop; one launch per call
    on either route."""
    obs, act, T, n = 17, 6, 60, 5
    dims, P, table, theta, spec = _problem(obs, (64, 64), act, T, scale=0.1)
    mean, std, clip = _norm(obs)
    idx = np.random.RandomState(4).randint(0, len(table) - P, size=n).astype(np.int64)
    assert eng.closed_mlp_plan([obs, 64, 64, act], spec.band) == (0, eng.sm_count, 0)
    coins = _coins(n, [(0, 0), (3, 1)])
    l0 = eng.launches
    new = _Run(eng, [obs, 64, 64, act], table, idx, theta, spec, mean, std, clip, sigma=0.05, coins=coins)
    assert eng.launches - l0 == 1
    old_fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
    old_behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
    osum, osq = (torch.zeros(obs, dtype=torch.float64, device=eng.device) for _ in range(2))
    ocnt = torch.zeros(2, dtype=torch.float64, device=eng.device)
    obs0, env_a, env_b = _dev_env(eng, spec)
    eng.rollout_closed(eng.to_device(table), eng.to_device(idx), eng.to_device(theta), 0.05, [obs, 64, 64, act], eng.to_device(mean),
                       eng.to_device(std), clip, obs0, env_a, env_b, eng.to_device(spec.rew_vec), spec.pos_scale, old_fit[0], old_fit[1],
                       1, old_behv[0].view(-1), old_behv[1].view(-1), coin_words=eng.to_device(coins.view(np.int32)),
                       save_obs_chance=0.5, ob_sum=osum, ob_sumsq=osq, ob_count=ocnt)
    eng.sync()
    assert np.array_equal(new.f, old_fit.cpu().numpy()) and np.array_equal(new.b, old_behv.cpu().numpy())
    assert np.array_equal(new.ocnt.cpu().numpy(), ocnt.cpu().numpy())
    assert np.allclose(new.osum.cpu().numpy(), osum.cpu().numpy(), rtol=1e-15, atol=0)    # (atomics: order of 2 terms)
    dims_w, P_w, table_w, theta_w, spec_w = _problem(15, (256, 256), 3, 10)
    l0 = eng.launches
    _Run(eng, [15, 256, 256, 3], table_w, [0, 5, 9], theta_w, spec_w, *_norm(15))
    assert eng.launches - l0 == 1


def test_closed_wide_bad_input(eng):
    from es_pytorch_b200._lib import EsLibraryError
    obs, act, T = 15, 3, 10
    dims, P, table, theta, spec = _problem(obs, (256, 256), act, T)
    mean, std, clip = _norm(obs)
    with pytest.raises(EsLibraryError):
        _Run(eng, [obs, 256, 256, act], table, [len(table) - P], theta, spec, mean, std, clip)   # idx + P == table length
    eng.sync()

    def refused(sizes, band=8, match=None):
        d = orc.layer_dims(sizes[0], sizes[1:-1], sizes[-1])
        Pn = orc.n_params(d)
        sp = orc.ClosedLoopEnvSpec(sizes[0], sizes[-1], T, band=band)
        with pytest.raises(EsLibraryError, match=match):
            eng.rollout_closed_mlp(eng.to_device(np.zeros(Pn + 10, np.float32)), torch.zeros(1, dtype=torch.int64, device=eng.device),
                                   eng.to_device(np.zeros(Pn, np.float32)), 0.02, sizes, eng.to_device(np.zeros(sizes[0])),
                                   eng.to_device(np.ones(sizes[0])), 5.0, *_dev_env(eng, sp), eng.to_device(sp.rew_vec), sp.pos_scale,
                                   torch.zeros(1, dtype=torch.float64, device=eng.device),
                                   torch.zeros(1, dtype=torch.float64, device=eng.device))
        with pytest.raises(EsLibraryError, match=match):
            eng.closed_mlp_plan(sizes, band)
    refused([17, 64, 64, 64, 64, 64, 6], match='2 to 4 hidden layers')
    refused([17, 256, 257, 6], match='hidden widths up to 256')
    refused([17, 256, 256, 65], match='act <= 64')
    refused([385, 64, 64, 6], match='obs <= 384')
    refused([17, 256, 256, 6], band=7, match='band must be even')
    refused([384, 256, 256, 256, 256, 64], band=16, match='bytes of shared memory per CTA in a cluster of 8 CTAs')


def _gen_args(eng, spec, table, theta, sizes, seeds, P, **kw):
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    return DeviceGeneration(eng.to_device(table), eng.to_device(theta.copy()), sizes, eng.to_device(spec.obs_stream),
                            eng.to_device(spec.rew_vec), [np.random.RandomState(s) for s in seeds], SIGMA, 0.005, Adam(P, 0.01),
                            coins_per_eval=1, engine=eng, closed=_dev_env(eng, spec), **kw)


def test_closed_wide_generation_matches_the_oracle(eng):
    """DeviceGeneration(closed=...) at 15-256-256-3: two generations, 2 streams x 4 pairs, save_obs coins, Adam -- indices and
    rank weights exact, fitness / theta / obs statistics to test_gpu_closed.py's tolerances."""
    obs, act, T = 15, 3, 50
    dims, P, table, theta, spec = _problem(obs, (256, 256), act, T)
    seeds = [500, 501]
    gen = _gen_args(eng, spec, table, theta, [obs, 256, 256, act], seeds, P, save_obs_chance=0.3)
    flat, opt = theta.copy(), orc.AdamOracle(P, 0.01)
    ostates = [np.random.RandomState(s) for s in seeds]
    z, o = np.zeros(obs), np.ones(obs)
    for g in range(2):
        th0 = flat.copy()
        st0 = [np.random.RandomState() for _ in seeds]
        for a, b in zip(st0, ostates):
            a.set_state(b.get_state())
        _assert_contractive(spec, orc.unflatten(th0, dims), z, o, 5.0)
        res = orc.generation(table, flat, opt, SIGMA, dims, spec, seeds, 4, z, o, 5.0, T, 500, 0.005, coins_per_eval=1,
                             rank_states=ostates)
        pos, neg, inds, _, obstat = orc.es_test_params(table, th0, SIGMA, dims, spec, seeds, 4, z, o, 5.0, T, coins_per_eval=1,
                                                       save_obs_chance=0.3, rank_states=st0)
        fpos, fneg = gen.evaluate(4)
        assert np.array_equal(gen.idx.cpu().numpy(), res['inds'].astype(np.int64))
        assert np.abs(fpos.cpu().numpy() - pos).max() <= 1e-4 and np.abs(fneg.cpu().numpy() - neg).max() <= 1e-4
        assert gen.gen_count.cpu().numpy()[0] == obstat.count and obstat.count > 0
        assert np.abs(gen.gen_sum.cpu().numpy() - obstat.sum).max() <= 1e-4 * max(1.0, np.abs(obstat.sum).max())
        assert np.abs(gen.gen_sumsq.cpu().numpy() - obstat.sumsq).max() <= 1e-4 * max(1.0, np.abs(obstat.sumsq).max())
        gen.update(fpos, fneg)
        assert np.array_equal(gen.weights.cpu().numpy(), res['weights'])
        assert np.abs(gen.theta.cpu().numpy() - flat).max() <= 3e-6
    fit0, _ = gen.noiseless_eval()                          # the noiseless evaluation of the updated theta, on the cluster kernel
    rews, _, _, _ = orc.run_model(spec, orc.unflatten(flat, dims), z, o, 5.0, T)
    assert abs(float(fit0[0]) - sum(rews)) <= 2e-5 * max(1.0, np.abs(rews).sum())


def test_closed_wide_generation_nsra(eng):
    """Two objectives at 15-256-256-3: the novelty column comes from the final positions the cluster kernel integrates."""
    obs, act, T = 15, 3, 30
    dims, P, table, theta, spec = _problem(obs, (256, 256), act, T)
    archive = np.random.RandomState(17).randn(12, 2) * 0.05
    seeds = [40, 41]
    gen = _gen_args(eng, spec, table, theta, [obs, 256, 256, act], seeds, P, archive=eng.to_device(archive, torch.float64),
                    nov_k=5, moo_w=0.5)
    fpos, fneg = gen.evaluate(4)
    pos, neg, inds, _, _ = orc.es_test_params(table, theta, SIGMA, dims, spec, seeds, 4, np.zeros(obs), np.ones(obs), 5.0, T,
                                              coins_per_eval=1, archive=archive, nov_k=5)
    assert np.array_equal(gen.idx.cpu().numpy(), inds.astype(np.int64))
    assert np.abs(fpos.cpu().numpy() - pos).max() <= 1e-4 and np.abs(fneg.cpu().numpy() - neg).max() <= 1e-4


def test_api_step_on_the_closed_loop_env_with_a_wide_policy(eng):
    """es.step with a BatchedRollout over ClosedLoopEnv(17, 6, T) and FeedForward([256, 256, 256]): two generations against
    orc.es_step, then the per-call fit_fn(policy.pheno(zeros), False) as one launch."""
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter

    class Cfg(dict):
        __getattr__ = dict.__getitem__
    obs, act, T, n = 17, 6, 45, 4
    hidden = (256, 256, 256)
    dims, P, table, theta, spec = _problem(obs, hidden, act, T)
    env = ClosedLoopEnv(obs, act, T)
    net = FeedForward(list(hidden), torch.nn.Tanh(), env, 0.0, 5)
    policy = Policy(net, SIGMA, Adam(P, 0.01))
    policy.flat_params[...] = theta
    policy.set_nn_params(policy.flat_params)
    nt = NoiseTable(P, table)
    seeds = [700, 701]
    streams, ref_streams = [np.random.RandomState(s) for s in seeds], [np.random.RandomState(s) for s in seeds]
    fit_fn = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.25, rank_streams=streams)
    cfg = Cfg(general=Cfg(policies_per_gen=2 * n, batch_size=500), policy=Cfg(l2coeff=0.005))
    ranker = CenteredRanker()
    assert es._can_fuse_step(dist.world(), policy, fit_fn, ranker)
    flat, opt = theta.copy(), orc.AdamOracle(P, 0.01)
    stat = orc.ObStatOracle((obs,), 1e-2)
    obmean, obstd = np.zeros(obs), np.ones(obs)
    for g in range(2):
        _assert_contractive(spec, orc.unflatten(flat, dims), obmean, obstd, 5.0)
        tr, gen_obstat = es.step(cfg, dist.world(), policy, nt, env, fit_fn, streams[0], ranker, Reporter())
        policy.update_obstat(gen_obstat)
        ref = orc.es_step(table, flat, opt, SIGMA, dims, spec, ref_streams, n, obmean, obstd, 5.0, T, 500, 0.005, coins_per_eval=1,
                          save_obs_chance=0.25, batched=False)
        stat.inc(ref['obstat'].sum, ref['obstat'].sumsq, ref['obstat'].count)
        obmean, obstd = stat.mean, stat.std
        assert np.array_equal(np.asarray(ranker.noise_inds), ref['inds'])
        tol = 1e-4 if g == 0 else 1e-3                  # (generation 1 normalises with the floored std: up to 10x gain)
        err = max(np.abs(ranker.fits_pos - ref['pos']).max(), np.abs(ranker.fits_neg - ref['neg']).max())
        assert err <= tol, (g, err)
        assert gen_obstat.count == ref['obstat'].count
        assert np.abs(gen_obstat.sum - ref['obstat'].sum).max() <= tol * max(1.0, np.abs(ref['obstat'].sum).max())
        if np.array_equal(ranker.ranked_fits, ref['weights']):
            assert np.abs(policy.flat_params - flat).max() <= 3e-6
        else:
            assert np.abs(policy.flat_params - flat).max() <= 1e-3
            policy.flat_params[...] = flat; policy.set_nn_params(policy.flat_params)
        assert abs(tr.result[0] - ref['noiseless'][0]) <= 10 * tol, (g, tr.result[0], ref['noiseless'][0])
        for a, b in zip(streams, ref_streams):
            assert np.array_equal(a.get_state()[1], b.get_state()[1]) and a.get_state()[2] == b.get_state()[2]
    l0 = eng.launches
    direct = fit_fn(policy.pheno(np.zeros(P)), False)
    assert eng.launches - l0 == 1
    for b in ref_streams:
        b.random()
    rews, _, _, _ = orc.run_model(spec, orc.unflatten(flat, dims), obmean, obstd, 5.0, T)
    assert abs(direct.result[0] - sum(rews)) <= 1e-3
