"""GPU parity of the CLOSED-LOOP synthetic env (SURVEY.md section 8d's optional variant, reported separately from the
open-loop headline): es_rollout_closedloop, a whole DeviceGeneration and es.step on it, against the oracle's literal
per-step loop (oracle.es_oracle.run_model).  float32 arithmetic in a different summation order than torch's
matrix-vector products: tolerances are stated per test; indices, coins and rank weights stay exact."""
import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu


def _problem(obs_dim, act_dim, T, seed=3, table_extra=120_000, scale=0.1, hidden=(64, 64), band=8):
    dims = orc.layer_dims(obs_dim, hidden, act_dim)
    P = orc.n_params(dims)
    rs = np.random.RandomState(seed)
    table = rs.randn(P + table_extra).astype(np.float32)
    theta = (rs.randn(P) * scale).astype(np.float32)
    return dims, P, table, theta, orc.ClosedLoopEnvSpec(obs_dim, act_dim, T, band=band)


def _dev_env(eng, spec):
    return (eng.to_device(spec.obs_stream[0].copy()), eng.to_device(np.ascontiguousarray(spec.env_a.T)),
            eng.to_device(np.ascontiguousarray(spec.env_b.T)))


@pytest.mark.parametrize('obs_dim,act_dim,T,n_pairs', [(17, 6, 60, 5), (376, 17, 40, 3), (24, 9, 33, 150), (100, 3, 25, 4)])
def test_closed_rollout_matches_the_oracle(eng, obs_dim, act_dim, T, n_pairs):
    """Fitness, final position and the ObStat increments of the saved rollouts, with a non-trivial observation
    normalisation (mean / std / an active clip)."""
    dims, P, table, theta, spec = _problem(obs_dim, act_dim, T)
    rs = np.random.RandomState(11)
    idx = rs.randint(0, len(table) - P, size=n_pairs).astype(np.int64)
    # (a normalisation that keeps the loop contractive: with std << 1 the map amplifies rounding differences -- chaos, where
    # no two float32 implementations agree -- so std is O(1) and the clip, which is active, small)
    mean, std, clip = rs.randn(obs_dim) * 0.05, 0.5 + rs.rand(obs_dim), 0.4
    coins = np.full((n_pairs, 4), 0xFFFFFFFF, dtype=np.uint32)
    saved = [(k, sgn) for k in range(n_pairs) for sgn in range(2) if (3 * k + sgn) % 4 == 0]
    for k, sgn in saved:
        coins[k, 2 * sgn:2 * sgn + 2] = 0                                           # u = 0 < chance
    obs0, env_a, env_b = _dev_env(eng, spec)
    fit = torch.zeros(2, n_pairs, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, n_pairs, 3, dtype=torch.float32, device=eng.device)
    osum, osq = (torch.zeros(obs_dim, dtype=torch.float64, device=eng.device) for _ in range(2))
    ocnt = torch.zeros(2, dtype=torch.float64, device=eng.device)
    eng.rollout_closed(eng.to_device(table), eng.to_device(idx), eng.to_device(theta), 0.05, [obs_dim, 64, 64, act_dim],
                       eng.to_device(mean), eng.to_device(std), clip, obs0, env_a, env_b, eng.to_device(spec.rew_vec), spec.pos_scale,
                       fit[0], fit[1], 1, behv[0].view(-1), behv[1].view(-1), coin_words=eng.to_device(coins.view(np.int32)),
                       save_obs_chance=0.5, ob_sum=osum, ob_sumsq=osq, ob_count=ocnt)
    eng.sync()
    got, gb = fit.cpu().numpy(), behv.cpu().numpy()
    check = range(n_pairs) if n_pairs <= 8 else [0, 1, n_pairs // 2, n_pairs - 2, n_pairs - 1]
    ref_sum, ref_sq = np.zeros(obs_dim), np.zeros(obs_dim)
    for k in check:
        for sgn, sign in enumerate((1.0, -1.0)):
            layers = orc.unflatten(orc.pheno_params(theta, 0.05, sign * orc.table_get(table, int(idx[k]), P)), dims)
            rews, bh, obs, _ = orc.run_model(spec, layers, mean, std, clip, T)
            want = orc.reward_result(rews)[0]
            assert abs(got[sgn, k] - want) <= 2e-5 * max(1.0, np.abs(rews).sum()), (k, sgn, got[sgn, k], want)
            assert np.abs(gb[sgn, k] - np.array(bh[-3:])).max() <= 1e-5
            if (k, sgn) in saved and n_pairs <= 8:
                ref_sum += obs.sum(axis=0).astype(np.float64)
                ref_sq += np.square(obs).sum(axis=0).astype(np.float64)
    assert ocnt.cpu().numpy().tolist() == [float(len(saved) * T), float(len(saved))]
    if n_pairs <= 8:
        assert np.abs(osum.cpu().numpy() - ref_sum).max() <= 1e-4 and np.abs(osq.cpu().numpy() - ref_sq).max() <= 1e-4


@pytest.mark.parametrize('obs_dim,act_dim,hidden,band', [(300, 40, (48, 24), 4), (384, 2, (64, 8), 16), (9, 33, (5, 64), 2)])
def test_closed_rollout_odd_shapes(eng, obs_dim, act_dim, hidden, band):
    """Shapes off the beaten path: more than 32 actions (two reward registers per lane), hidden layers that do not fill the
    thread rows, the widest / narrowest band, the largest observation; no ObStat buffers, no behaviour outputs."""
    T, n_pairs = 21, 3
    dims, P, table, theta, spec = _problem(obs_dim, act_dim, T, hidden=hidden, band=band)
    idx = np.random.RandomState(5).randint(0, len(table) - P, size=n_pairs).astype(np.int64)
    obs0, env_a, env_b = _dev_env(eng, spec)
    fit = torch.zeros(2, n_pairs, dtype=torch.float64, device=eng.device)
    eng.rollout_closed(eng.to_device(table), eng.to_device(idx), eng.to_device(theta), 0.05, [obs_dim, *hidden, act_dim],
                       eng.to_device(np.zeros(obs_dim)), eng.to_device(np.ones(obs_dim)), 5.0, obs0, env_a, env_b,
                       eng.to_device(spec.rew_vec), spec.pos_scale, fit[0], fit[1])
    eng.sync()
    got = fit.cpu().numpy()
    for k in range(n_pairs):
        for sgn, sign in enumerate((1.0, -1.0)):
            layers = orc.unflatten(orc.pheno_params(theta, 0.05, sign * orc.table_get(table, int(idx[k]), P)), dims)
            rews, _, _, _ = orc.run_model(spec, layers, np.zeros(obs_dim), np.ones(obs_dim), 5.0, T)
            assert abs(got[sgn, k] - sum(rews)) <= 2e-5 * max(1.0, np.abs(rews).sum()), (k, sgn, got[sgn, k], sum(rews))


def test_closed_generation_nsra(eng):
    """Two objectives on the closed-loop env: the novelty column comes from the final positions the kernel integrates."""
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    obs_dim, act_dim, T = 17, 6, 30
    dims, P, table, theta, spec = _problem(obs_dim, act_dim, T)
    archive = np.random.RandomState(17).randn(12, 2)
    seeds = [40, 41]
    gen = DeviceGeneration(eng.to_device(table), eng.to_device(theta.copy()), [obs_dim, 64, 64, act_dim], eng.to_device(spec.obs_stream),
                           eng.to_device(spec.rew_vec), [np.random.RandomState(s) for s in seeds], 0.05, 0.005, Adam(P, 0.01),
                           coins_per_eval=1, engine=eng, closed=_dev_env(eng, spec), archive=eng.to_device(archive, torch.float64),
                           nov_k=5, moo_w=0.5)
    fpos, fneg = gen.evaluate(4)
    pos, neg, inds, _, _ = orc.es_test_params(table, theta, 0.05, dims, spec, seeds, 4, np.zeros(obs_dim), np.ones(obs_dim), 5.0, T,
                                              coins_per_eval=1, archive=archive, nov_k=5)
    assert np.array_equal(gen.idx.cpu().numpy(), inds.astype(np.int64))
    assert np.abs(fpos.cpu().numpy() - pos).max() <= 1e-4 and np.abs(fneg.cpu().numpy() - neg).max() <= 1e-4


def test_closed_rollout_rejects_what_it_does_not_cover(eng):
    from es_pytorch_b200._lib import EsLibraryError
    dims, P, table, theta, spec = _problem(17, 6, 10)
    obs0, env_a, env_b = _dev_env(eng, spec)
    fit = torch.zeros(2, 1, dtype=torch.float64, device=eng.device)
    args = (0.05, [17, 64, 64, 6], eng.to_device(np.zeros(17)), eng.to_device(np.ones(17)), 5.0, obs0, env_a, env_b,
            eng.to_device(spec.rew_vec), spec.pos_scale, fit[0], fit[1])
    bad = torch.tensor([len(table)], dtype=torch.int64, device=eng.device)           # idx + P past the table: noisetable.py:34
    eng.rollout_closed(eng.to_device(table), bad, eng.to_device(theta), *args)
    with pytest.raises(EsLibraryError):
        eng.sync()
    dims3 = orc.layer_dims(17, (128, 64), 6)
    with pytest.raises(EsLibraryError):
        eng.rollout_closed(eng.to_device(np.zeros(orc.n_params(dims3) + 10, np.float32)), torch.zeros(1, dtype=torch.int64, device=eng.device),
                           eng.to_device(np.zeros(orc.n_params(dims3), np.float32)), 0.05, [17, 128, 64, 6], *args[2:])


def test_closed_generation_matches_the_oracle(eng):
    """DeviceGeneration(closed=...): two generations, 3 virtual ranks x 5 pairs, save_obs coins, Adam -- indices and rank
    weights exact, fitness / theta / obs statistics to float32 tolerance."""
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    obs_dim, act_dim, T = 24, 9, 50
    dims, P, table, theta, spec = _problem(obs_dim, act_dim, T)
    seeds = [500, 501, 502]
    gen = DeviceGeneration(eng.to_device(table), eng.to_device(theta.copy()), [obs_dim, 64, 64, act_dim], eng.to_device(spec.obs_stream),
                           eng.to_device(spec.rew_vec), [np.random.RandomState(s) for s in seeds], 0.05, 0.005, Adam(P, 0.01),
                           coins_per_eval=1, save_obs_chance=0.3, engine=eng, closed=_dev_env(eng, spec))
    flat, opt = theta.copy(), orc.AdamOracle(P, 0.01)
    ostates = [np.random.RandomState(s) for s in seeds]
    for g in range(2):
        th0 = flat.copy()
        st0 = [np.random.RandomState() for _ in seeds]
        for a, b in zip(st0, ostates):
            a.set_state(b.get_state())
        res = orc.generation(table, flat, opt, 0.05, dims, spec, seeds, 5, np.zeros(obs_dim), np.ones(obs_dim), 5.0, T, 500, 0.005,
                             coins_per_eval=1, rank_states=ostates)
        pos, neg, inds, _, obstat = orc.es_test_params(table, th0, 0.05, dims, spec, seeds, 5, np.zeros(obs_dim), np.ones(obs_dim), 5.0,
                                                       T, coins_per_eval=1, save_obs_chance=0.3, rank_states=st0)
        fpos, fneg = gen.evaluate(5)
        assert np.array_equal(gen.idx.cpu().numpy(), res['inds'].astype(np.int64))
        assert np.abs(fpos.cpu().numpy() - pos).max() <= 1e-4 and np.abs(fneg.cpu().numpy() - neg).max() <= 1e-4
        assert gen.gen_count.cpu().numpy()[0] == obstat.count and obstat.count > 0
        assert np.abs(gen.gen_sum.cpu().numpy() - obstat.sum).max() <= 1e-4 * max(1.0, np.abs(obstat.sum).max())
        assert np.abs(gen.gen_sumsq.cpu().numpy() - obstat.sumsq).max() <= 1e-4 * max(1.0, np.abs(obstat.sumsq).max())
        gen.update(fpos, fneg)
        assert np.array_equal(gen.weights.cpu().numpy(), res['weights'])
        assert np.abs(gen.theta.cpu().numpy() - flat).max() <= 3e-6


def test_closed_generation_refuses_action_noise(eng):
    from es_pytorch_b200.generation import DeviceGeneration
    from es_pytorch_b200.nn.optimizers import Adam
    dims, P, table, theta, spec = _problem(17, 6, 10)
    gen = DeviceGeneration(eng.to_device(table), eng.to_device(theta.copy()), [17, 64, 64, 6], eng.to_device(spec.obs_stream),
                           eng.to_device(spec.rew_vec), [np.random.RandomState(1)], 0.05, 0.005, Adam(P, 0.01), coins_per_eval=1,
                           engine=eng, closed=_dev_env(eng, spec), ac_std=0.01)
    with pytest.raises(NotImplementedError):
        gen.evaluate(2)


def test_api_step_on_the_closed_loop_env_matches_the_oracle(eng):
    """es.step (single-synchronisation route) with a BatchedRollout over ClosedLoopEnv: two generations incl. the ObStat
    update between them and the noiseless evaluation of the new theta."""
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
    obs_dim, act_dim, T, n = 17, 6, 45, 4
    dims, P, table, theta, spec = _problem(obs_dim, act_dim, T)
    env = ClosedLoopEnv(obs_dim, act_dim, T)
    assert np.array_equal(env.env_a, spec.env_a) and np.array_equal(env.env_b, spec.env_b) and np.array_equal(env.obs_stream, spec.obs_stream)
    net = FeedForward([64, 64], torch.nn.Tanh(), env, 0.0, 5)
    policy = Policy(net, 0.05, Adam(P, 0.01))
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
    stat = orc.ObStatOracle((obs_dim,), 1e-2)
    obmean, obstd = np.zeros(obs_dim), np.ones(obs_dim)
    for g in range(2):
        tr, gen_obstat = es.step(cfg, dist.world(), policy, nt, env, fit_fn, streams[0], ranker, Reporter())
        policy.update_obstat(gen_obstat)
        ref = orc.es_step(table, flat, opt, 0.05, dims, spec, ref_streams, n, obmean, obstd, 5.0, T, 500, 0.005, coins_per_eval=1,
                          save_obs_chance=0.25, batched=False)
        stat.inc(ref['obstat'].sum, ref['obstat'].sumsq, ref['obstat'].count)
        obmean, obstd = stat.mean, stat.std
        assert np.array_equal(np.asarray(ranker.noise_inds), ref['inds'])
        # generation 1 runs with the updated ObStat: std is floored at 0.1 (obstat.py:33), i.e. the normalisation multiplies the
        # observations (and every rounding difference in them) by up to 10 on each pass through the loop
        tol = 1e-4 if g == 0 else 1e-3
        err = max(np.abs(ranker.fits_pos - ref['pos']).max(), np.abs(ranker.fits_neg - ref['neg']).max())
        assert err <= tol, (g, err)
        assert gen_obstat.count == ref['obstat'].count
        assert np.abs(gen_obstat.sum - ref['obstat'].sum).max() <= tol * max(1.0, np.abs(ref['obstat'].sum).max())
        if np.array_equal(ranker.ranked_fits, ref['weights']):     # (a rank swap between near-equal fitnesses moves theta by more)
            assert np.abs(policy.flat_params - flat).max() <= 3e-6
        else:
            assert np.abs(policy.flat_params - flat).max() <= 1e-3
            policy.flat_params[...] = flat; policy.set_nn_params(policy.flat_params)
        assert abs(tr.result[0] - ref['noiseless'][0]) <= 10 * tol, (g, tr.result[0], ref['noiseless'][0])
        for a, b in zip(streams, ref_streams):
            assert np.array_equal(a.get_state()[1], b.get_state()[1]) and a.get_state()[2] == b.get_state()[2]
    # the per-policy route (an opaque call of the fit_fn) runs the same episode as one launch
    direct = fit_fn(policy.pheno(np.zeros(P)), False)
    for b in ref_streams:
        b.random()
    layers = orc.unflatten(flat, dims)
    rews, _, _, _ = orc.run_model(spec, layers, obmean, obstd, 5.0, T)
    assert abs(direct.result[0] - sum(rews)) <= 1e-3
