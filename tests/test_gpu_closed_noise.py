"""GPU: closed-loop rollouts with action noise and multi-episode evaluations (es_rollout_closedloop_mlp_episodes) against the
oracle's literal per-step loop (oracle.es_oracle.run_model), on the one-CTA kernel (rollout_closed.cu) and the cluster kernel
(rollout_closedw.cu), plus DeviceGeneration, es.step and the per-call fit_fn on top of them.

The kernels add float32(gaussian * ac_std) to the float32 action in float32; the reference adds the float64 product and rounds
once, so an action may differ by one float32 ulp.  Every case is first checked to be contractive under its noise, so those
differences stay at rounding size; the bounds are test_gpu_closed_wide.py's."""
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
    rs = np.random.RandomState(seed)
    return rs.randn(obs) * 0.05, 0.5 + rs.rand(obs), 0.4


def _dev_env(eng, spec):
    return (eng.to_device(spec.obs_stream[0].copy()), eng.to_device(np.ascontiguousarray(spec.env_a.T)),
            eng.to_device(np.ascontiguousarray(spec.env_b.T)))


def _layers(theta, table, idx, P, dims, sign):
    return orc.unflatten(orc.pheno_params(theta, SIGMA, sign * orc.table_get(table, int(idx), P)), dims)


def _coins(n, saved):
    coins = np.full((n, 4), 0xFFFFFFFF, dtype=np.uint32)
    for k, sgn in saved:
        coins[k, 2 * sgn:2 * sgn + 2] = 0                                           # u = 0 < chance
    return coins


def _gauss(k, sgn, E, T, act):
    """The gaussians of evaluation (k, sgn): one stream per evaluation, drawn as the reference draws them."""
    return np.random.RandomState(1000 + 2 * k + sgn).randn(E * T * act)


def _assert_contractive(spec, layers, mean, std, clip, ac_std, steps=150):
    s = orc.ClosedLoopEnvSpec(spec.obs_dim, spec.act_dim, steps, band=spec.band)
    _, _, a, _ = orc.run_model(s, layers, mean, std, clip, steps, ac_std=ac_std, rs=np.random.RandomState(5))
    s.obs_stream = s.obs_stream.copy()
    s.obs_stream[0] += np.float32(0.3)
    _, _, b, _ = orc.run_model(s, layers, mean, std, clip, steps, ac_std=ac_std, rs=np.random.RandomState(5))
    assert np.abs(a[-1] - b[-1]).max() < 1e-6, 'the loop is not contractive under this noise: the comparison would mean nothing'


class _Run:
    """One rollout_closed_mlp call with every output: fit [2][n], behv [2][n][3], ObStat sums and counts."""

    def __init__(self, eng, sizes, table, idx, theta, spec, mean, std, clip, noise=None, E=1, coins=None):
        n, obs = len(idx), sizes[0]
        self.fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
        self.behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
        self.osum, self.osq = (torch.zeros(obs, dtype=torch.float64, device=eng.device) for _ in range(2))
        self.ocnt = torch.zeros(2, dtype=torch.float64, device=eng.device)
        obs0, env_a, env_b = _dev_env(eng, spec)
        l0 = eng.launches
        eng.rollout_closed_mlp(eng.to_device(table), eng.to_device(np.asarray(idx, np.int64)), eng.to_device(theta), SIGMA, sizes,
                               eng.to_device(mean), eng.to_device(std), clip, obs0, env_a, env_b, eng.to_device(spec.rew_vec),
                               spec.pos_scale, self.fit[0], self.fit[1], 1, self.behv[0].view(-1), self.behv[1].view(-1),
                               coin_words=None if coins is None else eng.to_device(coins.view(np.int32)), save_obs_chance=0.5,
                               ob_sum=self.osum, ob_sumsq=self.osq, ob_count=self.ocnt,
                               act_noise=None if noise is None else eng.to_device(np.ascontiguousarray(noise, np.float32)),
                               episodes=E)
        eng.sync()
        self.launches = eng.launches - l0
        self.f, self.b = self.fit.cpu().numpy(), self.behv.cpu().numpy()
        self.stats = (self.osum.cpu().numpy(), self.osq.cpu().numpy(), self.ocnt.cpu().numpy())

    def same(self, other, stats=True):
        return (np.array_equal(self.f, other.f) and np.array_equal(self.b, other.b)
                and (not stats or all(np.array_equal(a, b) for a, b in zip(self.stats, other.stats))))


# two hidden layers <= 64 (the one-CTA kernel) and every shipped cluster shape
SHAPES = [
    ('17-64-64-6', 17, (64, 64), 6, 60),
    ('376-64-64-17', 376, (64, 64), 17, 40),
    ('simple_conf', 15, (256, 256), 3, 60),
    ('obj', 17, (256, 256, 256), 6, 40),
    ('ns', 28, (256, 256, 256), 8, 40),
    ('flagrun', 28, (128, 256, 256, 128), 8, 40),
]


@pytest.mark.parametrize('E', [1, 2, 10])
@pytest.mark.parametrize('ac_std', [0.01, 0.05])
@pytest.mark.parametrize('name,obs,hidden,act,T', SHAPES, ids=[s[0] for s in SHAPES])
def test_noisy_closed_rollout_matches_the_oracle(eng, name, obs, hidden, act, T, ac_std, E):
    """Fitness (the per-step mean over E episodes), the last episode's final position and the ObStat of the saved
    evaluations (from the last episode), with one kernel launch."""
    dims, P, table, theta, spec = _problem(obs, hidden, act, T)
    mean, std, clip = _norm(obs)
    n = 2
    idx = np.random.RandomState(7).randint(0, len(table) - P, size=n).astype(np.int64)
    _assert_contractive(spec, _layers(theta, table, idx[0], P, dims, 1.0), mean, std, clip, ac_std)
    sizes = [obs, *hidden, act]
    assert (eng.closed_mlp_plan(sizes, spec.band)[0] == 0) == (hidden == (64, 64))
    saved = [(0, 0), (1, 1)]
    noise = np.stack([np.stack([(_gauss(k, s, E, T, act) * ac_std).astype(np.float32) for s in range(2)]) for k in range(n)])
    run = _Run(eng, sizes, table, idx, theta, spec, mean, std, clip, noise, E, _coins(n, saved))
    assert run.launches == 1
    ref_sum, ref_sq = np.zeros(obs), np.zeros(obs)
    for k in range(n):
        for sgn, sign in enumerate((1.0, -1.0)):
            rews, bh, ob, _ = orc.run_model(spec, _layers(theta, table, idx[k], P, dims, sign), mean, std, clip, T, ac_std=ac_std,
                                            rs=np.random.RandomState(1000 + 2 * k + sgn), episodes=E)
            want = sum(rews)
            assert abs(run.f[sgn, k] - want) <= 2e-5 * max(1.0, np.abs(rews).sum()), (k, sgn, run.f[sgn, k], want)
            pos_tol = max(1e-5, T * float(np.spacing(np.float32(np.abs(bh[-3:]).max()))))
            assert np.abs(run.b[sgn, k] - np.array(bh[-3:])).max() <= pos_tol, (k, sgn)
            if (k, sgn) in saved:
                ref_sum += ob.sum(axis=0).astype(np.float64)
                ref_sq += np.square(ob).sum(axis=0).astype(np.float64)
    assert run.stats[2].tolist() == [2.0 * T, 2.0]
    assert np.abs(run.stats[0] - ref_sum).max() <= 1e-4 and np.abs(run.stats[1] - ref_sq).max() <= 1e-4


EDGE = [('17-64-64-6', 17, (64, 64), 6, 30), ('simple_conf', 15, (256, 256), 3, 30), ('flagrun', 28, (128, 256, 256, 128), 8, 30)]


@pytest.mark.parametrize('name,obs,hidden,act,T', EDGE, ids=[s[0] for s in EDGE])
def test_noisy_closed_rollout_bit_exact_edges(eng, name, obs, hidden, act, T):
    """No noise (any E) and all-zero noise give the noise-free rollout; two equal episodes give one; an episode after a
    different one starts afresh (behaviour and ObStat are the last episode's alone)."""
    dims, P, table, theta, spec = _problem(obs, hidden, act, T)
    mean, std, clip = _norm(obs)
    n = 3
    idx = np.random.RandomState(9).randint(0, len(table) - P, size=n).astype(np.int64)
    sizes, coins = [obs, *hidden, act], _coins(n, [(0, 0), (1, 1), (2, 0), (2, 1)])
    args = (eng, sizes, table, idx, theta, spec, mean, std, clip)
    base = _Run(*args, coins=coins)
    for E in (1, 3):
        assert _Run(*args, None, E, coins).same(base)
        assert _Run(*args, np.zeros((n, 2, E * T * act), np.float32), E, coins).same(base)
    rs = np.random.RandomState(4)
    n0 = (rs.randn(n, 2, 1, T * act) * 0.05).astype(np.float32)
    n1 = (rs.randn(n, 2, 1, T * act) * 0.05).astype(np.float32)
    one = _Run(*args, n0.reshape(n, 2, -1), 1, coins)
    assert not one.same(base, stats=False)
    assert _Run(*args, np.concatenate([n0, n0], axis=2).reshape(n, 2, -1), 2, coins).same(one)
    mixed = _Run(*args, np.concatenate([n1, n0], axis=2).reshape(n, 2, -1), 2, coins)
    assert np.array_equal(mixed.b, one.b) and all(np.array_equal(a, b) for a, b in zip(mixed.stats, one.stats))
    assert not np.array_equal(mixed.f, one.f)


def test_binned_head_refuses_action_noise(eng):
    from es_pytorch_b200.nn.nn import BinnedHead
    obs, T, adim, bins = 17, 10, 3, 4
    dims, P, table, theta, spec = _problem(obs, (64, 64), adim * bins, T)
    spec = orc.ClosedLoopEnvSpec(obs, adim, T)
    head = BinnedHead(bins, np.full(adim, -1.0, np.float32), np.full(adim, 1.0, np.float32))
    obs0, env_a, env_b = _dev_env(eng, spec)
    fit = torch.zeros(2, 1, dtype=torch.float64, device=eng.device)
    with pytest.raises(ValueError):
        eng.rollout_closed_mlp(eng.to_device(table), torch.zeros(1, dtype=torch.int64, device=eng.device), eng.to_device(theta), SIGMA,
                               [obs, 64, 64, adim * bins], eng.to_device(np.zeros(obs)), eng.to_device(np.ones(obs)), 5.0, obs0,
                               env_a, env_b, eng.to_device(spec.rew_vec), spec.pos_scale, fit[0], fit[1], head=head,
                               act_noise=torch.zeros(2 * T * adim, dtype=torch.float32, device=eng.device))


@pytest.mark.parametrize('E', [1, 3])
def test_device_generation_with_closed_action_noise_matches_the_oracle(eng, E):
    """Two generations, ac_std = 0.01, 3 virtual ranks, one save_obs coin per evaluation: indices and coins exact, the
    stream state exact (the cached gaussian to 1 ulp), fitness within 1e-4, ObStat, rank weights and theta as in
    test_gpu_closed.py."""
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    obs, act, T, n, ac_std = 24, 9, 31, 4, 0.01                      # T * act odd: the gaussian cache crosses evaluations
    dims, P, table, theta, spec = _problem(obs, (64, 64), act, T, scale=0.1, table_extra=120_000)
    seeds = [500, 501, 502]
    streams, ref = [np.random.RandomState(s) for s in seeds], [np.random.RandomState(s) for s in seeds]
    streams[1].randn(1); ref[1].randn(1)
    gen = DeviceGeneration(eng.to_device(table), eng.to_device(theta.copy()), [obs, 64, 64, act], eng.to_device(spec.obs_stream),
                           eng.to_device(spec.rew_vec), streams, 0.05, 0.005, Adam(P, 0.01), coins_per_eval=1, save_obs_chance=0.3,
                           engine=eng, closed=_dev_env(eng, spec), ac_std=ac_std, episodes=E, closed_act_noise=True)
    flat, opt = theta.copy(), orc.AdamOracle(P, 0.01)
    for g in range(2):
        th0 = flat.copy()
        st0 = [np.random.RandomState() for _ in seeds]
        for a, b in zip(st0, ref):
            a.set_state(b.get_state())
        res = orc.generation(table, flat, opt, 0.05, dims, spec, [None] * 3, n, np.zeros(obs), np.ones(obs), 5.0, T, 500, 0.005,
                             coins_per_eval=1, rank_states=ref, save_obs_chance=0.3, ac_std=ac_std, episodes=E)
        fpos, fneg = gen.evaluate(n)
        assert np.array_equal(gen.idx.cpu().numpy(), res['inds'].astype(np.int64))
        assert np.abs(fpos.cpu().numpy() - res['pos']).max() <= 1e-4 and np.abs(fneg.cpu().numpy() - res['neg']).max() <= 1e-4
        ob = res['obstat']
        assert gen.gen_count.cpu().numpy()[0] == ob.count
        assert np.abs(gen.gen_sum.cpu().numpy() - ob.sum).max() <= 1e-4 * max(1.0, np.abs(ob.sum).max())
        assert np.abs(gen.gen_sumsq.cpu().numpy() - ob.sumsq).max() <= 1e-4 * max(1.0, np.abs(ob.sumsq).max())
        for a, b in zip(gen.rank_states(), ref):
            sa, sb = a.get_state(), b.get_state()
            assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2] and sa[3] == sb[3], f'stream after generation {g}'
            assert abs(sa[4] - sb[4]) <= np.spacing(abs(sb[4]))
        gen.update(fpos, fneg)
        assert np.array_equal(gen.weights.cpu().numpy(), res['weights'])
        assert np.abs(gen.theta.cpu().numpy() - flat).max() <= 1e-5


class _Cfg(dict):
    __getattr__ = dict.__getitem__


@pytest.mark.parametrize('width,E', [(64, 1), (64, 3), (256, 2)])
def test_es_step_with_closed_action_noise_matches_the_oracle(eng, width, E):
    """es.step (fused: one synchronisation) with BatchedRollout(ClosedLoopEnv, episodes=E) and FeedForward(ac_std=0.01),
    ac_std decayed between the two generations as obj.py:81 does; then the per-call fit_fn with use_ac_noise=True as one
    launch."""
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
    obs, act, T, n = 17, 6, 33, 4
    hidden = (width, width)
    dims, P, table, theta, spec = _problem(obs, hidden, act, T, scale=0.05 if width == 64 else 0.03, table_extra=120_000)
    env = ClosedLoopEnv(obs, act, T)
    net = FeedForward(list(hidden), torch.nn.Tanh(), env, 0.01, 5)
    policy = Policy(net, 0.05, Adam(P, 0.01))
    policy.flat_params[...] = theta
    policy.set_nn_params(policy.flat_params)
    nt = NoiseTable(P, table)
    seeds = [700, 701]
    streams, ref_streams = [np.random.RandomState(s) for s in seeds], [np.random.RandomState(s) for s in seeds]
    fit_fn = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.25, rank_streams=streams, episodes=E)
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))
    ranker = CenteredRanker()
    assert es._can_fuse_step(dist.world(), policy, fit_fn, ranker)
    flat, opt = theta.copy(), orc.AdamOracle(P, 0.01)
    ac_std = 0.01
    for g in range(2):
        tr, _ = es.step(cfg, dist.world(), policy, nt, env, fit_fn, streams[0], ranker, Reporter())
        ref = orc.es_step(table, flat, opt, 0.05, dims, spec, ref_streams, n, np.zeros(obs), np.ones(obs), 5.0, T, 500, 0.005,
                          coins_per_eval=1, save_obs_chance=0.25, batched=False, ac_std=ac_std, episodes=E)
        assert np.array_equal(np.asarray(ranker.noise_inds), ref['inds'])
        err = max(np.abs(ranker.fits_pos - ref['pos']).max(), np.abs(ranker.fits_neg - ref['neg']).max())
        assert err <= 1e-4, (g, err)
        if np.array_equal(ranker.ranked_fits, ref['weights']):
            assert np.abs(policy.flat_params - flat).max() <= 1e-5
        else:                                                       # a rank swap between near-equal fitnesses
            assert np.abs(policy.flat_params - flat).max() <= 1e-3
            policy.flat_params[...] = flat; policy.set_nn_params(policy.flat_params)
        assert abs(tr.result[0] - ref['noiseless'][0]) <= 1e-3
        for a, b in zip(streams, ref_streams):
            sa, sb = a.get_state(), b.get_state()
            assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2] and sa[3] == sb[3] and abs(sa[4] - sb[4]) <= np.spacing(abs(sb[4]))
        ac_std *= 0.5                                               # obj.py:81
        net._action_std = ac_std
    # the per-call route with noise: one launch, the first stream advanced as the reference's fit_fn advances it
    l0 = eng.launches
    direct = fit_fn(policy.pheno(np.zeros(P)), True)
    assert eng.launches - l0 == 1
    for b in ref_streams:
        b.random()
    rews, _, _, _ = orc.run_model(spec, orc.unflatten(flat, dims), np.zeros(obs), np.ones(obs), 5.0, T, ac_std=ac_std,
                                  rs=ref_streams[0], episodes=E)
    assert abs(direct.result[0] - sum(rews)) <= 1e-4
    for a, b in zip(streams, ref_streams):
        sa, sb = a.get_state(), b.get_state()
        assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2] and sa[3] == sb[3] and abs(sa[4] - sb[4]) <= np.spacing(abs(sb[4]))
