"""GPU: multi-episode evaluations (obj.py:54-63, ``eps_per_policy``): es_rollout_openloop_episodes against the episode
oracle, E = 1 against es_rollout_openloop_noisy, the tensor-core modes against float32, DeviceGeneration and es.step."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu


def dev(eng, a):
    return eng.to_device(np.ascontiguousarray(a))


class _Replay:
    """Stands in for the RandomState of run_model: ``randn(act)`` returns the next row of a pre-drawn noise array."""

    def __init__(self, a):
        self.a, self.i = a.astype(np.float64), 0

    def randn(self, n):
        self.i += 1
        return self.a[self.i - 1]


def _problem(eng, obs, hidden, act, T, n_pairs, E, seed):
    rs = np.random.RandomState(seed)
    dims = orc.layer_dims(obs, hidden, act)
    P = orc.n_params(dims)
    L = P + 200_000
    table, theta = rs.randn(L).astype(np.float32), (rs.randn(P) * 0.1).astype(np.float32)
    idx = rs.randint(0, L - P - 1, size=n_pairs).astype(np.int64)
    env = orc.SyntheticEnvSpec(obs, act, T)
    noise = (rs.randn(n_pairs, 2, E, T, act) * 0.05).astype(np.float32)
    obsn = eng.normalise_obs(dev(eng, env.obs_stream[:T]), dev(eng, np.zeros(obs)), dev(eng, np.ones(obs)), 5.0)
    return dict(dims=dims, P=P, table=table, theta=theta, idx=idx, env=env, noise=noise, obsn=obsn,
                sizes=[obs] + list(hidden) + [act], T=T, n=n_pairs)


def _run(eng, pb, mode, noise, E):
    n = pb['n']
    fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
    eng.rollout(dev(eng, pb['table']), dev(eng, pb['idx']), dev(eng, pb['theta']), 0.02, pb['sizes'], pb['obsn'],
                dev(eng, pb['env'].rew_vec), pb['env'].pos_scale, fit[0], fit[1], 1, behv[0], behv[1], mode,
                act_noise=None if noise is None else dev(eng, noise), episodes=E)
    eng.sync()
    return fit.cpu().numpy(), behv.cpu().numpy()


# obs, hidden, act, T, n_pairs: the packed-FMA kernel (two shapes), the general kernel with the weights in a global scratch,
# and a few pairs (the general kernel splitting the episode's time tiles over the SMs)
SHAPES = [(17, (64, 64), 6, 150, 80), (376, (64, 64), 17, 60, 80), (15, (256, 256), 3, 70, 70), (17, (64, 64), 6, 150, 3)]


@pytest.mark.parametrize('E', [1, 2, 3, 7])
@pytest.mark.parametrize('shape', SHAPES, ids=['17-64-64-6', '376-64-64-17', '15-256-256-3', 'few-pairs'])
def test_f32_episodes_match_the_oracle(eng, shape, E):
    obs, hidden, act, T, n = shape
    pb = _problem(eng, obs, hidden, act, T, n, E, seed=obs + T + E)
    f, b = _run(eng, pb, 0, pb['noise'], E)
    for k in sorted({0, 1, n // 2, n - 1}):
        eps = orc.table_get(pb['table'], int(pb['idx'][k]), pb['P'])
        for s, nz in ((0, eps), (1, -eps)):
            layers = orc.unflatten(orc.pheno_params(pb['theta'], 0.02, nz), pb['dims'])
            rews, bb, _, _ = orc.run_model(pb['env'], layers, np.zeros(obs), np.ones(obs), 5.0, T, True, ac_std=1.0,
                                           rs=_Replay(pb['noise'][k, s].reshape(E * T, act)), episodes=E)
            assert abs(f[s, k] - orc.reward_result(rews)[0]) <= 1e-5 * max(1.0, np.abs(rews).sum()), (k, s)
            assert np.allclose(b[s, k], bb[-3:], rtol=1e-4, atol=1e-5), (k, s)          # the last episode's position


def _noisy_direct(eng, pb, mode, noise):
    """es_rollout_openloop_noisy called directly (the single-episode entry point)."""
    n = pb['n']
    fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
    table, idx, theta = dev(eng, pb['table']), dev(eng, pb['idx']), dev(eng, pb['theta'])
    rew, nz = dev(eng, pb['env'].rew_vec), dev(eng, noise)
    if mode != 0:
        eng.lib.es_noise_table_changed(eng._ctx)
    ls = (C.c_int * 4)(*pb['sizes'])
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = eng.lib.es_rollout_openloop_noisy(eng._ctx, p(table), table.numel(), p(idx), n, p(theta), theta.numel(), 0.02, ls, 3,
                                           p(pb['obsn']), p(rew), pb['T'], pb['env'].pos_scale, p(fit[0]), p(fit[1]), 1,
                                           p(behv[0]), p(behv[1]), p(nz), mode, eng.stream)
    assert rc == 0
    eng.sync()
    return fit.cpu().numpy(), behv.cpu().numpy()


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('n_pairs', [9, 160])
def test_one_episode_is_the_noisy_rollout_bit_for_bit(eng, mode, n_pairs):
    pb = _problem(eng, 24, (64, 64), 9, 130, n_pairs, 1, seed=5 + n_pairs)
    f1, b1 = _run(eng, pb, mode, pb['noise'], 1)
    f0, b0 = _noisy_direct(eng, pb, mode, pb['noise'])
    assert np.array_equal(f1, f0) and np.array_equal(b1, b0)


@pytest.mark.parametrize('mode', [1, 2])
@pytest.mark.parametrize('E', [2, 5])
def test_tensor_core_episodes_match_f32(eng, mode, E):
    """The per-mode tolerances test_rollout_with_action_noise applies against the float32 kernel."""
    T = 130
    pb = _problem(eng, 24, (64, 64), 9, T, 160, E, seed=11 + E)
    f, b = _run(eng, pb, mode, pb['noise'], E)
    f32, b32 = _run(eng, pb, 0, pb['noise'], E)
    f1, _ = _run(eng, pb, 0, np.ascontiguousarray(pb['noise'][:, :, -1:]), 1)
    assert np.abs(f32 - f1).max() > 1e-3, 'the episodes must change the fitness'
    spread = max(f32.std(), 1e-3 * np.sqrt(T))
    tol = 6e-6 if mode == 2 else 5e-3
    assert np.sqrt(((f - f32) ** 2).mean()) <= tol * spread + (1e-6 if mode == 2 else 2e-4)
    assert np.abs(b - b32).max() <= (2e-6 if mode == 2 else 2e-3) * 0.05 * T + 1e-4


def test_noiseless_episodes_are_one_episode(eng):
    """Without action noise the entry point treats any episode count as one episode (bit for bit)."""
    pb = _problem(eng, 17, (64, 64), 6, 90, 80, 1, seed=3)
    f1, b1 = _run(eng, pb, 0, None, 1)
    f5, b5 = _run(eng, pb, 0, None, 5)
    assert np.array_equal(f1, f5) and np.array_equal(b1, b5)


@pytest.mark.parametrize('jump', [None, '1'])
def test_device_generation_episodes_match_the_oracle(eng, monkeypatch, jump):
    """Two generations, ac_std = 0.01, 3 episodes, 3 virtual ranks, one save_obs coin per evaluation: per evaluation the coin,
    then 3 x T x act gaussians back to back in the stream.  Indices, obs statistics (the coins decide them) and the stream
    state (key, position, has_gauss) exact, the cached gaussian to 2 ulp; rank weights exact; fitness and theta to float32
    tolerance.
    ES_MT_JUMP=1 forces the jump-ahead draw."""
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    if jump is not None:
        monkeypatch.setenv('ES_MT_JUMP', jump)
    obs, act, hidden, T, n, E, ac_std = 17, 5, (64, 64), 37, 4, 3, 0.01    # T * act odd: the cache crosses episodes
    dims = orc.layer_dims(obs, hidden, act)
    P = orc.n_params(dims)
    rs0 = np.random.RandomState(8)
    table, theta = rs0.randn(P + 150_000).astype(np.float32), (rs0.randn(P) * 0.1).astype(np.float32)
    env = orc.SyntheticEnvSpec(obs, act, T)
    seeds = [300, 301, 302]
    streams = [np.random.RandomState(s) for s in seeds]
    ref = [np.random.RandomState(s) for s in seeds]
    streams[1].randn(1); ref[1].randn(1)
    gen = DeviceGeneration(eng.to_device(table), eng.to_device(theta.copy()), [obs, 64, 64, act], eng.to_device(env.obs_stream),
                           eng.to_device(env.rew_vec), streams, 0.02, 0.005, Adam(P, 0.01), ob_clip=5.0,
                           pos_scale=env.pos_scale, engine=eng, coins_per_eval=1, save_obs_chance=0.4, ac_std=ac_std,
                           episodes=E)
    flat, opt = theta.copy(), orc.AdamOracle(P, 0.01)
    for g in range(2):
        fpos, fneg = gen.evaluate(n)
        gen.update(fpos, fneg)
        res = orc.generation(table, flat, opt, 0.02, dims, env, [None] * 3, n, np.zeros(obs), np.ones(obs), 5.0, T, 500, 0.005,
                             coins_per_eval=1, rank_states=ref, save_obs_chance=0.4, ac_std=ac_std, episodes=E)
        assert np.array_equal(gen.idx.cpu().numpy(), res['inds'].astype(np.int64))
        assert np.abs(fpos.cpu().numpy()[:, 0] - res['pos'][:, 0]).max() <= 1e-4
        assert np.abs(fneg.cpu().numpy()[:, 0] - res['neg'][:, 0]).max() <= 1e-4
        assert np.array_equal(gen.weights.cpu().numpy(), res['weights'])                # rank weights bit-exact
        # theta after Adam: the reconstructed gradient differs from numpy's dot in its last bits, and Adam divides by
        # sqrt(v), which magnifies that on the near-zero components (3.99e-6 measured on an H100, steps of 0.01)
        assert np.abs(gen.theta.cpu().numpy() - flat).max() <= 1e-5
        ob = res['obstat']
        assert gen.gen_count.cpu().numpy()[0] == ob.count
        assert np.array_equal(gen.gen_sum.cpu().numpy(), ob.sum) and np.array_equal(gen.gen_sumsq.cpu().numpy(), ob.sumsq)
        for a, b in zip(gen.rank_states(), ref):
            sa, sb = a.get_state(), b.get_state()
            assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2] and sa[3] == sb[3], f'stream after generation {g}'
            assert abs(sa[4] - sb[4]) <= 2 * np.spacing(abs(sb[4]))


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _api_objects(table, theta, spec, hidden):
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    env = SyntheticEnv(spec.obs_dim, spec.act_dim, spec.T)
    net = FeedForward(list(hidden), torch.nn.Tanh(), env, 0.0, 5)
    policy = Policy(net, 0.02, Adam(len(theta), 0.01))
    policy.flat_params[...] = theta
    policy.set_nn_params(policy.flat_params)
    return env, net, policy, NoiseTable(len(theta), table)


def test_es_step_episodes_fused_matches_call_by_call(eng):
    """es.step with BatchedRollout(episodes=3) on the fused route against the same kind of object behind an opaque callable
    (es.test_params' per-perturbation loop, every evaluation one launch of all 3 episodes): indices, fitness, theta and the
    stream state agree over two generations."""
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    obs, act, hidden, T, n, E = 17, 5, (64, 64), 37, 4, 3
    spec = orc.SyntheticEnvSpec(obs, act, T)
    P = orc.n_params(orc.layer_dims(obs, hidden, act))
    rs0 = np.random.RandomState(12)
    table, theta = rs0.randn(P + 150_000).astype(np.float32), (rs0.randn(P) * 0.1).astype(np.float32)
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))
    runs = []
    for fused in (True, False):
        env, net, policy, nt = _api_objects(table, theta.copy(), spec, hidden)
        net._action_std = 0.01
        rs = np.random.RandomState(99)
        rs.randn(1)
        bro = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.25, rank_streams=[rs], episodes=E)
        fit_fn = bro if fused else (lambda model, use_ac_noise=True, f=bro: f(model, use_ac_noise))
        ranker = CenteredRanker()
        assert es._can_fuse_step(dist.world(), policy, fit_fn, ranker) == fused
        out = []
        for g in range(2):
            tr, _ = es.step(cfg, dist.world(), policy, nt, env, fit_fn, rs, ranker, Reporter())
            out.append((np.asarray(ranker.noise_inds).copy(), np.asarray(ranker.fits_pos).copy(),
                        np.asarray(ranker.fits_neg).copy(), policy.flat_params.copy(), rs.get_state(), tr.result[0]))
        runs.append(out)
    for (ia, pa, na, ta, sa, ra), (ib, pb, nb, tb, sb, rb) in zip(*runs):
        assert np.array_equal(ia, ib)
        assert np.abs(pa - pb).max() <= 1e-4 and np.abs(na - nb).max() <= 1e-4
        assert np.abs(ta - tb).max() <= 3e-6
        assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2] and sa[3] == sb[3] and abs(sa[4] - sb[4]) <= 2 * np.spacing(abs(sb[4]))
        assert abs(ra - rb) <= 1e-4
