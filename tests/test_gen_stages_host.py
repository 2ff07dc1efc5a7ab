"""CPU: the stage-by-stage generation judge (tests/gen_stages.py) on generations of the oracle (oracle.es_oracle.generation)
standing in for the device's, and the modelled pipeline bugs it must reject.

The captured generation is the second of two on the same streams and optimizer (3 streams x 7 pairs, 17-64-64-6, T = 48, one
save_obs coin per evaluation at chance 0.3, Adam), so Adam's state, the streams' state and the observation statistics are
carried over and the normalisation runs with the first generation's mean / std.  Variants: NSRA (a 16-entry archive, k = 10,
w = 0.5) and action noise (ac_std = 0.01).  The oracle computes its rollouts in float32 on the CPU, so the fitness is judged
with the float32 rollout's bounds (ES_ROLLOUT_F32); gsum is the oracle's own numpy reconstruction (es_oracle.scale_noise).
The oracle's policies are tanh stacks: the activation variants ('activation': leaky ReLU of slope 0.1 on the plain capture;
'closed_activation': ELU of alpha 0.7 on the closed-loop one) take the oracle's generation with its fitness replaced by the
float64 truth of the activation (and, in the closed loop, the ObStat sums by the truth's), everything after it rescored.
The oracle does not hand out the raw coin words it drew, so the captured words (and the action noise) are the judge's own replay
of the streams: on the host the coin-word check compares the replay with itself, and what ties the oracle's coins to the judge
is the obs statistics (count and n_saved from the oracle's rs.random() calls) and the streams' end states.  The
'+ coin on the - evaluation' bug is rejected here by that word check alone.
"""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_stages as gs  # noqa: E402
import rc_f64 as rc  # noqa: E402
from oracle import es_oracle as orc  # noqa: E402

F32 = np.float32
MODE_F32 = 0                    # _lib.ES_ROLLOUT_F32
SIZES, T, SEEDS, N_PER = [17, 64, 64, 6], 48, (1000, 1001, 1002), 7
CHANCE, LR, SIGMA, L2 = 0.3, 0.01, 0.02, 0.005
# rank shifts against the float64 truth at 42 evaluations: the oracle's float32 fitness is within ~1e-7 of the spread
SHIFT_BOUND, DW_BOUND = 1, 1.0 / 41


def _state(rs):
    st = rs.get_state()
    return (st[1].copy(), int(st[2]), int(st[3]), float(st[4]))


def _capture(variant):
    """Variants: 'plain', 'nsra' (16-entry archive, w = 0.5), 'noise' (ac_std 0.01), 'episodes' (E = 3, ac_std 0.01),
    'nsr' (a 5-entry archive with k = 10, w = 0.25) and 'closed' (the closed-loop env, theta of scale 1 / sqrt(fan_in) as
    test_gpu_closed_f64's init regime)."""
    archive = {'nsra': np.random.RandomState(17).randn(16, 2), 'nsr': np.random.RandomState(18).randn(5, 2)}.get(variant)
    moo_w = {'nsra': 0.5, 'nsr': 0.25}.get(variant)
    ac_std = 0.01 if variant in ('noise', 'episodes') else 0.0
    episodes = 3 if variant == 'episodes' else 1
    closed = variant == 'closed'
    dims = orc.layer_dims(SIZES[0], SIZES[1:-1], SIZES[-1])
    P = orc.n_params(dims)
    rs0 = np.random.RandomState(5)
    table = rs0.randn(P + 20_000).astype(F32)
    theta = (rs0.randn(P) * 0.1).astype(F32)
    if closed:
        theta = np.concatenate([rs0.randn(fi * fo + fo) / np.sqrt(fi) for fi, fo in zip(SIZES[:-1], SIZES[1:])]).astype(F32)
    # closed loop: the first generation's statistics give std ~0.1, which amplifies the normalised observations ten-fold; at
    # b_gain 0.1 a 1e-9 move of obs_0 grows 0.6-fold over the episode (at the default 0.5: 1.2e3-fold, chaotic)
    env = orc.ClosedLoopEnvSpec(SIZES[0], SIZES[-1], T, b_gain=0.1) if closed else orc.SyntheticEnvSpec(SIZES[0], SIZES[-1], T)
    streams = [np.random.RandomState(s) for s in SEEDS]
    opt = orc.AdamOracle(P, LR)
    kw = dict(coins_per_eval=1, rank_states=streams, save_obs_chance=CHANCE, ac_std=ac_std, archive=archive, nov_k=10,
              moo_w=moo_w, episodes=episodes)
    obmean, obstd = np.zeros(SIZES[0]), np.ones(SIZES[0])
    g1 = orc.generation(table, theta, opt, SIGMA, dims, env, [None] * 3, N_PER, obmean, obstd, 5.0, T, 500, L2, **kw)
    stat = orc.ObStatOracle((SIZES[0],), 1e-2)                   # Policy.update_obstat's running statistics
    stat.inc(g1['obstat'].sum, g1['obstat'].sumsq, g1['obstat'].count)
    obmean, obstd = stat.mean, stat.std
    theta0, m0, v0, t0 = theta.copy(), opt.m.copy(), opt.v.copy(), opt.t
    streams0 = [_state(rs) for rs in streams]
    g2 = orc.generation(table, theta, opt, SIGMA, dims, env, [None] * 3, N_PER, obmean, obstd, 5.0, T, 500, L2, **kw)
    idx = g2['inds'].astype(np.int64)
    K = len(idx)
    w = np.asarray(g2['weights'], dtype=F32).reshape(-1)
    gsum = np.asarray(orc.scale_noise(w, idx, table, P, 500), dtype=F32)
    ob = g2['obstat']
    stats = np.concatenate([ob.sum, ob.sumsq, [float(ob.count), float(ob.count) / T]])
    behv = None
    if archive is not None:                                     # the final positions the oracle's novelty was computed from
        behv = np.zeros((2, K, 3), dtype=F32)
        for k in range(K):
            for s, sign in enumerate((1.0, -1.0)):
                layers = orc.unflatten(orc.pheno_params(theta0, SIGMA, sign * table[idx[k]:idx[k] + P]), dims)
                _, b, _, _ = orc.run_model(env, layers, obmean, obstd, 5.0, T, batched=True)
                behv[s, k] = b[-3:]
    cap = gs.Capture(sizes=SIZES, T=T, sigma=SIGMA, l2coeff=L2, ob_clip=5.0, pos_scale=env.pos_scale, save_obs_chance=CHANCE,
                     ac_std=ac_std, lr=LR, table=torch.from_numpy(table), obs_stream=env.obs_stream, rew_vec=env.rew_vec,
                     theta0=theta0, m0=m0, v0=v0, t0=t0, streams0=streams0, ob_mean=obmean, ob_std=obstd, idx=idx,
                     coin_words=np.zeros((K, 4), dtype=np.uint32),
                     obsn=None if closed else orc.normalise_obs(env.obs_stream[:T], obmean, obstd, 5.0),
                     fit=np.stack([g2['pos'], g2['neg']]), stats=stats, weights=w, n_ranked=g2['n_ranked'], gsum=gsum,
                     theta1=theta.copy(), m1=opt.m.copy(), v1=opt.v.copy(), t1=opt.t, streams1=[_state(rs) for rs in streams],
                     behv=behv, archive=archive, episodes=episodes, **({'moo_w': moo_w} if archive is not None else {}))
    if closed:
        cap.obs0, cap.band = env.obs_stream[0].copy(), env.band
        cap.env_a, cap.env_b = np.ascontiguousarray(env.env_a.T), np.ascontiguousarray(env.env_b.T)
    # the coin words and the action noise: the streams' draws between the indices, in the order the oracle consumed them
    noise = []
    for r in range(len(SEEDS)):
        _, words, _, nz = gs.replay_stream(cap, r)
        cap.coin_words[r * N_PER:(r + 1) * N_PER] = words
        if ac_std:
            noise.append(nz.astype(F32))
    if ac_std:
        cap.act_noise = np.concatenate(noise)
    return cap


def _activation_capture(base, act):
    """``base``'s capture for a policy with activation ``act``: the fitness that policy earns (the float64 truth), the
    closed loop's ObStat sums of its saved evaluations, and everything after the fitness rescored."""
    cap = gs._copy(_cap(base), activation=act)
    f = cap.fit.copy()
    if cap.closed:
        cap = gs._closed_saved_sums(cap)
        f[:, :, 0] = gs.closed_truth(cap, pairs=range(cap.K), growth=False)['fit']
    else:
        f[:, :, 0] = gs.fitness_truth(cap)[0]
    return gs._rescored(gs._copy(cap, fit=f))


def _act(kind, param):
    from es_pytorch_b200 import _lib
    from es_pytorch_b200.nn.nn import Activation
    return Activation(getattr(_lib, kind), float(np.float32(param)))


_CAPS = {}


def _cap(variant):
    if variant not in _CAPS:
        if variant == 'activation':
            _CAPS[variant] = _activation_capture('plain', _act('ES_ACT_LEAKY_RELU', 0.1))
        elif variant == 'closed_activation':
            _CAPS[variant] = _activation_capture('closed', _act('ES_ACT_ELU', 0.7))
        else:
            _CAPS[variant] = _capture(variant)
    return _CAPS[variant]


def _judge(cap):
    return gs.judge(cap, MODE_F32, rc.H100_SMS, SHIFT_BOUND, DW_BOUND, tie=list(range(cap.K)))


@pytest.mark.parametrize('variant', ['plain', 'nsra', 'noise', 'episodes', 'nsr', 'closed', 'activation', 'closed_activation'])
def test_judge_passes_the_oracle_generation(variant):
    cap = _cap(variant)
    checks = _judge(cap)
    print('\n' + gs.report(f'oracle generation, {variant}', checks))
    gs.assert_ok(checks)
    assert cap.extra['n_saved'] > 0 and cap.t0 == 1
    assert not np.array_equal(cap.ob_std, np.ones_like(cap.ob_std))
    if variant.startswith('closed'):              # every saved evaluation in the truth's sample, the whole population here
        assert len(cap.extra['closed_truth']['pairs']) == cap.K and cap.extra['ranks_vs_truth'].startswith('not compared')


def _variant(name):
    """The capture a modelled bug is judged on: the 'nsr' capture has w = 0.25 and 5 archive entries for k = 10."""
    need = gs.NEEDS.get(name, 'nsra' if name in gs.NEEDS_ARCHIVE else 'plain')
    return 'activation' if need == 'param' else need


@pytest.mark.parametrize('name', sorted(gs.MUTATIONS))
def test_judge_rejects_modelled_bugs(name):
    what, mutate = gs.MUTATIONS[name]
    cap = _cap(_variant(name))
    checks = _judge(mutate(cap))
    stages, margin = gs.rejection(checks)
    print(f'\n{name} ({what}): rejected by {stages}, margin {margin:.3g}x')
    assert stages is not None, f'{what}: not rejected'
    assert margin >= 10, (what, stages, margin)


@pytest.mark.parametrize('name', gs.ACT_MUTATIONS)
def test_judge_rejects_activation_bugs_in_the_closed_loop(name):
    what, mutate = gs.MUTATIONS[name]
    cap = _cap('closed_activation')
    _judge(cap)                                   # leaves the truth's sample in cap.extra, as the GPU files judge first
    stages, margin = gs.rejection(_judge(mutate(cap)))
    print(f'\n{name} ({what}), closed loop: rejected by {stages}, margin {margin:.3g}x')
    assert stages is not None and margin >= 10, (what, stages, margin)


def test_activation_of_tanh_is_the_tanh_truth():
    """A capture whose activation is tanh gets the truths of one without (no activation): open loop with episodes and
    action noise, closed loop with its growth, to 1e-13 relative; and the closed loop's truth with another activation is
    closed_f64.truth's of the sampled pairs, sliced from the table by hand."""
    import closed_f64
    import f64_rollout
    tanh = _act('ES_ACT_TANH', 0.0)
    cap = _cap('episodes')
    for want, got in zip(gs.fitness_truth(cap), gs.fitness_truth(gs._copy(cap, activation=tanh))):
        np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-300)
    cap = _cap('closed')
    want, got = gs.closed_truth(cap), gs.closed_truth(gs._copy(cap, activation=tanh))
    for k in ('fit', 'mass', 'behv', 'mag', 'osum', 'osq', 'oabs'):
        np.testing.assert_allclose(got[k], want[k], rtol=1e-13, atol=1e-300, err_msg=k)
    assert abs(got['growth'] - want['growth']) <= 1e-13 * want['growth']
    elu = _act('ES_ACT_ELU', 0.7)
    c = gs._copy(cap, activation=elu)
    got = gs.closed_truth(c, growth=False)
    pairs = got['pairs']
    P = c.P
    table = np.concatenate([c.table[int(c.idx[k]):int(c.idx[k]) + P].numpy() for k in pairs])
    want = closed_f64.truth(table, np.arange(len(pairs)) * P, c.theta0, c.sigma, c.sizes, c.ob_mean, c.ob_std, c.ob_clip,
                            c.obs0, c.env_a, c.env_b, c.rew_vec, c.pos_scale, activation=f64_rollout.elu(0.7))
    for k in ('fit', 'mass', 'behv', 'mag', 'osum', 'osq', 'oabs'):     # sums in another order: relative to their largest
        np.testing.assert_allclose(got[k], want[k], rtol=1e-13, atol=1e-13 * np.abs(want[k]).max(), err_msg=k)
    assert not np.allclose(got['fit'], gs.closed_truth(cap, pairs=pairs, growth=False)['fit'])
