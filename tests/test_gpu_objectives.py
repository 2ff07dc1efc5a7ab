"""GPU: the single-objective adaptors (MeanRewardResult, DistResult, XDistResult, NSResult) on the device.

* es_fitness_objective at the C ABI against the host classes' own get_result, bit for bit, on edge-case numbers.
* es.step through BatchedRollout(result=X) against an opaque fit_fn written as the reference's scripts write one
  (rs.random(), run_model, X(rews, behv, obs, steps)), same seeds and streams, two generations, on every fused route.
* NSResult's column against NSRResult's novelty column; a cached generation switched between objectives; two processes.

Tolerances, per route (R on an episode total, Q on a final coordinate):
  * open loop F32 and with action noise (E = 3): R = 1e-4, the existing call-by-call tests' fitness bound
    (test_gpu_episodes.py); Q = T float32 ulps of the position (per-step float32 sums, tile order vs step order);
  * binned F32: the same decisions, so R = 1e-12 of the reward mass and Q as above (test_gpu_binned.py);
  * TC3: the mode's outputs are within ~1e-6 of float64 (test_gpu_binned.py, test_gpu_generation.py), so a step's reward is
    within 1e-6 * sum_j |c_tj| and R = 2e-6 * sum_t,j |c_tj|; a coordinate is pos_scale * sum_t a_t, so
    Q = 2e-6 * pos_scale * T + T float32 ulps;
  * closed loop (one-CTA and cluster kernels): R = 2e-5 of the reward mass, Q = max(1e-5, T ulps) (test_gpu_closed_wide.py).
A mean reward is within R / (T - 1); a distance and a novelty are 1-Lipschitz in (x, y), within sqrt(2) Q; a final x within Q.
"""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LOW = np.array([-0.3, -1.0, 0.1], dtype=np.float32)
HIGH = np.array([2.7, 1.0, 0.35], dtype=np.float32)


def _classes():
    from es_pytorch_b200.gym import training_result as tr
    return tr.MeanRewardResult, tr.DistResult, tr.XDistResult, tr.NSResult


# ------------------------------------------------------------------------------------------------------------- the kernel
def _edge_numbers(n, seed=0):
    """float64 totals and float32 positions over many magnitudes, with +-0, subnormals and values near 2^+-60."""
    rs = np.random.RandomState(seed)
    tot = rs.randn(n) * np.exp2(rs.randint(-70, 70, n).astype(np.float64))
    special_t = np.array([0.0, -0.0, 5e-324, -5e-324, 2.0 ** -1030, 2.0 ** 60, -2.0 ** 60, 2.0 ** -60, 1.0, -1.0,
                          np.nextafter(2.0 ** 60, 0), 3.0 ** 38, 1e308, -1e308])
    tot[:len(special_t)] = special_t
    pos = (rs.randn(n, 3) * np.exp2(rs.randint(-70, 70, (n, 3)).astype(np.float64))).astype(np.float32)
    f32 = np.float32
    special_p = np.array([[0.0, 0.0, 1.0], [-0.0, -0.0, 0.0], [-0.0, 0.0, 2.0], [1e-45, -1e-45, 0.0], [1e-40, 3e-39, 0.0],
                          [2.0 ** 60, 2.0 ** 60, 0.0], [-2.0 ** 60, 2.0 ** -60, 0.0], [2.0 ** -60, -2.0 ** -60, 0.0],
                          [3.4e38, 3.4e38, 0.0], [-3.4e38, 1.0, 0.0], [np.finfo(f32).tiny, -np.finfo(f32).tiny, 0.0],
                          [1.0, 0.0, 0.0], [-3.0, 4.0, 0.0], [1.5, -2.5e-3, 7.0]], dtype=f32)
    pos[:len(special_p)] = special_p
    # a share of positions where x and y have very different magnitudes, and one where they are equal
    pos[n // 2:n // 2 + 100, 1] = pos[n // 2:n // 2 + 100, 0] * np.float32(2.0 ** -30)
    pos[n // 2 + 100:n // 2 + 200, 1] = pos[n // 2 + 100:n // 2 + 200, 0]
    return tot, pos


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


@pytest.mark.parametrize('steps', [1, 2, 7, 999, 2 ** 31 - 1])
def test_objective_kernel_is_the_host_classes_bit_for_bit(eng, steps):
    from es_pytorch_b200 import _lib
    Mean, Dist, XDist, _ = _classes()
    n = 3000
    tot, pos = _edge_numbers(n, seed=steps % 1000)
    behv = eng.to_device(np.ascontiguousarray(pos))
    no_obs = np.zeros((1, 4))
    for kind, cls in ((_lib.ES_OBJ_MEAN_REWARD, Mean), (_lib.ES_OBJ_DIST, Dist), (_lib.ES_OBJ_XDIST, XDist)):
        # stride 2, as the NSRA layout: the other column is left as it was
        fit = np.stack((tot, np.arange(n, dtype=np.float64) + 0.5), axis=1)
        dfit = eng.to_device(np.ascontiguousarray(fit))
        eng.fitness_objective(kind, dfit.view(-1), 2, behv if cls is not Mean else None, n, steps)
        got = dfit.cpu().numpy()
        want = np.array([cls([float(tot[e])], [float(v) for v in pos[e]], no_obs, steps).result[0] for e in range(n)],
                        dtype=np.float64)
        # (the reference's reward is sum([total]), which starts from 0: a -0.0 total has a +0.0 mean)
        bad = np.nonzero(_bits(got[:, 0]) != _bits(want))[0]
        assert bad.size == 0, (cls.__name__, steps, [(tot[e], pos[e], got[e, 0], want[e]) for e in bad[:5]])
        assert np.array_equal(got[:, 1], fit[:, 1])


def test_objective_kernel_refusals(eng):
    from es_pytorch_b200 import _lib
    fit = torch.zeros(8, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(8, 3, dtype=torch.float32, device=eng.device)
    with pytest.raises(_lib.EsLibraryError, match='steps = 0'):
        eng.fitness_objective(_lib.ES_OBJ_MEAN_REWARD, fit, 1, None, 8, 0)
    with pytest.raises(_lib.EsLibraryError, match='unknown kind'):
        eng.fitness_objective(0, fit, 1, behv, 8, 5)
    with pytest.raises(_lib.EsLibraryError, match='NULL'):
        eng.fitness_objective(_lib.ES_OBJ_DIST, fit, 1, None, 8, 5)
    l0 = eng.launches
    eng.fitness_objective(_lib.ES_OBJ_XDIST, fit, 1, behv, 0, 5)       # nothing to do: no launch
    eng.fitness_objective(_lib.ES_OBJ_XDIST, fit, 1, behv, 8, 5)
    assert eng.launches - l0 == 1


# ---------------------------------------------------------------------------------------------------------- every route
class _Cfg(dict):
    __getattr__ = dict.__getitem__


ROUTES = {
    # name: (closed, obs, hidden, act, T, n pairs, rollout mode, binned, ac_std, episodes)
    'f32': (False, 32, (64, 64), 6, 24, 8, 'f32', False, 0.0, 1),
    'tc3': (False, 32, (64, 64), 6, 24, 8, 'tc3', False, 0.0, 1),
    'binned': (False, 15, (64, 64), 3, 24, 8, 'f32', True, 0.0, 1),
    'noise_e3': (False, 17, (64, 64), 5, 37, 4, 'f32', False, 0.01, 3),
    'closed_64': (True, 17, (64, 64), 6, 24, 6, 'f32', False, 0.0, 1),
    'closed_256': (True, 15, (256, 256), 3, 24, 6, 'f32', False, 0.0, 1),
}


def _tolerances(route, env, T, pos_abs):
    ulps = T * float(np.spacing(np.float32(max(pos_abs, 1e-30))))
    mass = float(np.abs(env.rew_vec[:T]).sum())
    if route in ('f32', 'noise_e3'):
        return 1e-4, max(1e-7, ulps)
    if route == 'binned':
        return 1e-12 * max(1.0, 3.0 * mass), max(1e-7, ulps)
    if route == 'tc3':
        return 2e-6 * mass, 2e-6 * env.pos_scale * T + ulps
    return 2e-5 * max(1.0, mass), max(1e-5, ulps)


def _objective_tol(cls, R, Q, T):
    Mean, Dist, XDist, NS = _classes()
    return {Mean: R / (T - 1), Dist: np.sqrt(2) * Q, XDist: Q, NS: np.sqrt(2) * Q}[cls]


class _Record:
    """A reporter that keeps what es.step reports per generation: the noiseless result and the summed steps."""

    def __init__(self):
        self.steps, self.noiseless = [], []

    def print(self, *a, **k):
        pass

    def log(self, *a, **k):
        pass

    def log_gen(self, fits, noiseless_tr, policy, steps):
        self.steps.append(int(steps))
        self.noiseless.append(noiseless_tr.result[0])


def _run_route(route, cls, archive=None, gens=2):
    from es_pytorch_b200 import _lib, dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    from es_pytorch_b200.gym.training_result import NSResult
    from es_pytorch_b200.nn.nn import FeedForward, FFBinned
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker
    closed, obs, hidden, act, T, n, mode, binned, ac_std, E = ROUTES[route]
    env = (ClosedLoopEnv if closed else SyntheticEnv)(obs, act, T)
    if binned:
        env.action_space.low, env.action_space.high = LOW[:act].copy(), HIGH[:act].copy()
    nets = [FFBinned(list(hidden), torch.nn.Tanh(), env, 5, 5) if binned else
            FeedForward(list(hidden), torch.nn.Tanh(), env, ac_std, 5) for _ in range(2)]
    P = len(Policy.get_flat(nets[0]))
    rs0 = np.random.RandomState(21)
    table = rs0.randn(P + 50_000).astype(np.float32)
    theta = (rs0.randn(P) * (0.1 if not closed else 0.05)).astype(np.float32)
    policies = []
    for net in nets:
        p = Policy(net, 0.02, Adam(P, 0.01))
        p.flat_params[...] = theta
        p.set_nn_params(p.flat_params)
        policies.append(p)
    nts = [NoiseTable(P, table.copy()) for _ in range(2)]
    streams = [np.random.RandomState(77), np.random.RandomState(77)]
    if ac_std:
        streams[0].randn(1); streams[1].randn(1)            # both start with a cached gaussian
    chance = 0.25
    cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n, batch_size=500), policy=_Cfg(l2coeff=0.005))
    rollout_mode = {'f32': _lib.ES_ROLLOUT_F32, 'tc3': _lib.ES_ROLLOUT_TC3}[mode]
    fused = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=chance, archive=archive, nov_k=5, rollout_mode=rollout_mode,
                           episodes=E, result=cls)
    zeros = np.array([np.zeros(env.observation_space.shape)])

    def opaque(model, use_ac_noise=True):               # the scripts' fit_fn (obj.py:54-63, nsra.py:89-94)
        rs = streams[1]
        save_obs = rs.random() < chance
        rews = np.zeros(T)
        for _ in range(max(1, E)):
            rew, behv, obs_, steps = run_model(model, env, T, rs if use_ac_noise else None)
            rews[:len(rew)] += np.array(rew)
        rews /= max(1, E)
        o = obs_ if save_obs else zeros
        if cls is NSResult:
            return cls(rews.tolist(), behv[-3:], o, steps, archive, 5)
        return cls(rews.tolist(), behv, o, steps)

    rankers = [CenteredRanker(), CenteredRanker()]
    assert es._can_fuse_step(dist.world(), policies[0], fused, rankers[0])
    assert not es._can_fuse_step(dist.world(), policies[1], opaque, rankers[1])
    recs = [_Record(), _Record()]
    out = []
    for g in range(gens):
        res = []
        for p, nt, fit_fn, st, rk, rec in zip(policies, nts, (fused, opaque), streams, rankers, recs):
            es.step(cfg, dist.world(), p, nt, env, fit_fn, st, rk, rec)
            res.append(dict(inds=np.asarray(rk.noise_inds).copy(), w=np.asarray(rk.ranked_fits).copy(),
                            fits=np.concatenate((np.asarray(rk.fits_pos), np.asarray(rk.fits_neg))).ravel(),
                            theta=p.flat_params.copy(), state=st.get_state(), steps=rec.steps[-1], noiseless=rec.noiseless[-1]))
        out.append(res)
    return out, env, T


def _pos_bound(route):
    T = ROUTES[route][4]
    return 0.05 * T * (3.0 if ROUTES[route][7] else 1.0)            # |a| <= 1 (tanh) or <= 3 (the binned bounds)


def _assert_same(out, cls, route, env, T):
    R, Q = _tolerances(route, env, T, _pos_bound(route))
    tol = _objective_tol(cls, R, Q, T)
    for g, (a, b) in enumerate(out):
        assert np.array_equal(a['inds'], b['inds']), g
        sa, sb = a['state'], b['state']
        assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2] and sa[3] == sb[3], g
        assert abs(sa[4] - sb[4]) <= 2 * np.spacing(abs(sb[4])), g
        assert a['steps'] == b['steps'] == 2 * len(a['inds']) * (T - 1), (g, a['steps'], b['steps'])
        err = np.abs(a['fits'] - b['fits']).max()
        assert err <= tol, (g, cls.__name__, route, err, tol)
        assert abs(a['noiseless'] - b['noiseless']) <= tol, (g, a['noiseless'], b['noiseless'], tol)
        # the same ranks wherever the reference's objectives are further apart than the bound allows a swap
        srt = np.sort(b['fits'])
        if np.diff(srt).min() > 2 * tol:
            assert np.array_equal(a['w'], b['w']), g
            assert np.abs(a['theta'] - b['theta']).max() <= 3e-6, (g, np.abs(a['theta'] - b['theta']).max())


@pytest.mark.parametrize('route', list(ROUTES))
@pytest.mark.parametrize('name', ['MeanRewardResult', 'DistResult', 'XDistResult', 'NSResult'])
def test_es_step_fused_objective_matches_the_scripts_fit_fn(eng, route, name):
    Mean, Dist, XDist, NS = _classes()
    cls = {c.__name__: c for c in (Mean, Dist, XDist, NS)}[name]
    archive = None
    if cls is NS:
        if ROUTES[route][9] > 1:
            pytest.skip('no reference script averages episodes for novelty search (BatchedRollout refuses it)')
        archive = np.random.RandomState(17).randn(12, 2) * 0.3
    out, env, T = _run_route(route, cls, archive)
    _assert_same(out, cls, route, env, T)
    if cls is not Mean:                                      # the objective separates the evaluations
        assert not np.allclose(out[0][0]['fits'], out[0][0]['fits'][0])


# ------------------------------------------------------------------------------------------------- NSResult, cache, multi
def _objects(env, theta_seed=5):
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    net = FeedForward([64, 64], torch.nn.Tanh(), env, 0.0, 5)
    P = len(Policy.get_flat(net))
    rs0 = np.random.RandomState(theta_seed)
    table, theta = rs0.randn(P + 40_000).astype(np.float32), (rs0.randn(P) * 0.1).astype(np.float32)
    policy = Policy(net, 0.02, Adam(P, 0.01))
    policy.flat_params[...] = theta
    policy.set_nn_params(policy.flat_params)
    return policy, NoiseTable(P, table)


def _test_params(fit_fn, objs, seed, n=6):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.nn.obstat import ObStat
    policy, nt = objs
    return es.test_params(dist.world(), n, policy, nt, ObStat(fit_fn.env.observation_space.shape, 0), fit_fn,
                          np.random.RandomState(seed))


@pytest.mark.parametrize('closed', [False, True])
def test_ns_result_column_is_the_nsr_novelty_column(eng, closed):
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    from es_pytorch_b200.gym.training_result import NSResult, NSRResult
    env = (ClosedLoopEnv if closed else SyntheticEnv)(17, 6, 30)
    archive = np.random.RandomState(4).randn(9, 2) * 0.2
    objs = _objects(env)
    ns = _test_params(BatchedRollout(env, 30, archive=archive, nov_k=4, result=NSResult), objs, 8)
    nsr = _test_params(BatchedRollout(env, 30, archive=archive, nov_k=4, result=NSRResult), objs, 8)
    assert ns[0].shape == (6, 1) and nsr[0].shape == (6, 2)
    assert np.array_equal(ns[2], nsr[2]) and ns[3] == nsr[3]
    assert np.array_equal(_bits(ns[0][:, 0]), _bits(nsr[0][:, 1])) and np.array_equal(_bits(ns[1][:, 0]), _bits(nsr[1][:, 1]))


def test_cached_generation_switched_between_objectives_is_a_fresh_one(eng):
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
    from es_pytorch_b200.gym.training_result import DistResult, MeanRewardResult, RewardResult, XDistResult
    env = SyntheticEnv(17, 6, 30)
    objs = _objects(env)
    prev = BatchedRollout(env, 30, result=RewardResult)
    _test_params(prev, objs, 3)
    for cls in (DistResult, MeanRewardResult, XDistResult, RewardResult, XDistResult):
        switched = BatchedRollout(env, 30, result=cls)
        switched._gen = prev._gen                          # a generation cached for another objective
        got = _test_params(switched, objs, 11)
        assert switched._gen is not prev._gen and switched._gen.objective == switched.objective
        fresh = _test_params(BatchedRollout(env, 30, result=cls), objs, 11)
        for a, b in zip(got[:3], fresh[:3]):
            assert np.array_equal(_bits(a), _bits(b)), cls.__name__
        kept = switched._gen
        again = _test_params(switched, objs, 11)           # same objective: the cached generation is kept
        assert switched._gen is kept
        for a, b in zip(again[:3], fresh[:3]):
            assert np.array_equal(_bits(a), _bits(b)), cls.__name__
        prev = switched


_MULTI_WORKER = '''
import os, sys
sys.path.insert(0, {root!r})
import numpy as np, torch
from es_pytorch_b200 import dist
from es_pytorch_b200.core import es
from es_pytorch_b200.core.noisetable import NoiseTable
from es_pytorch_b200.core.policy import Policy
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.gym.batched import BatchedRollout
from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
from es_pytorch_b200.gym.training_result import DistResult
from es_pytorch_b200.nn.nn import FeedForward
from es_pytorch_b200.nn.optimizers import Adam
from es_pytorch_b200.utils.rankers import CenteredRanker
from es_pytorch_b200.utils.reporters import Reporter
multi = 'LOCAL_RANK' in os.environ
comm = dist.init_from_env('nccl') if multi else dist.world()
eng = get_engine(int(os.environ.get('LOCAL_RANK', 0)))
obs_dim, act_dim, T, n = 17, 6, 48, 10
env = SyntheticEnv(obs_dim, act_dim, T)
net = FeedForward([64, 64], torch.nn.Tanh(), env, 0.0, 5)
P = len(Policy.get_flat(net))
rs = np.random.RandomState(0)
table = rs.randn(P + 200_000).astype(np.float32); theta = (rs.randn(P) * 0.1).astype(np.float32)
policy = Policy(net, 0.02, Adam(P, 0.01)); policy.flat_params[...] = theta; policy.set_nn_params(policy.flat_params)
nt = NoiseTable(P, table)
seeds = [1000 + 2 * r for r in range(4)]                        # 4 ranks: 2 per process, or all 4 in one
per = 4 // comm.size
streams = [np.random.RandomState(s) for s in seeds[per * comm.rank: per * comm.rank + per]]
fit_fn = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.2, rank_streams=streams, result=DistResult)
class C(dict): __getattr__ = dict.__getitem__
cfg = C(general=C(policies_per_gen=2 * n * comm.size, batch_size=500), policy=C(l2coeff=0.005))
ranker = CenteredRanker()
assert es._can_fuse_step(comm, policy, fit_fn, ranker)
out = {{}}
for g in range(2):
    es.step(cfg, comm, policy, nt, env, fit_fn, streams[0], ranker, Reporter())
    out['inds%d' % g] = np.asarray(ranker.noise_inds); out['w%d' % g] = np.asarray(ranker.ranked_fits)
    out['pos%d' % g] = np.asarray(ranker.fits_pos); out['neg%d' % g] = np.asarray(ranker.fits_neg)
    out['theta%d' % g] = policy.flat_params.copy()
if comm.rank == 0:
    np.savez(sys.argv[1], **out)
os.write(1, ('DIST_OK_%d\\n' % comm.rank).encode())
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpu_dist_result_matches_one_process(tmp_path):
    """DistResult through es.step on two processes (2 virtual ranks each) against one process carrying all 4 ranks, within
    test_gpu_multi.py's tolerances."""
    script = tmp_path / 'wd.py'
    script.write_text(_MULTI_WORKER.format(root=ROOT))
    one = subprocess.run([sys.executable, str(script), str(tmp_path / 'one.npz')], capture_output=True, text=True, timeout=600)
    assert one.returncode == 0, (one.stdout + one.stderr)[-3000:]
    with socket.socket() as sk:
        sk.bind(('127.0.0.1', 0))
        port = sk.getsockname()[1]
    two = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr',
                          '127.0.0.1', '--master-port', str(port), str(script), str(tmp_path / 'two.npz')],
                         capture_output=True, text=True, timeout=600)
    assert two.returncode == 0, (two.stdout + two.stderr)[-3000:]
    assert 'DIST_OK_0' in two.stdout and 'DIST_OK_1' in two.stdout
    a, b = np.load(tmp_path / 'one.npz'), np.load(tmp_path / 'two.npz')
    for g in range(2):
        assert np.array_equal(a['inds%d' % g], b['inds%d' % g])
        assert np.abs(a['pos%d' % g] - b['pos%d' % g]).max() < 1e-3 and np.abs(a['neg%d' % g] - b['neg%d' % g]).max() < 1e-3
        assert np.array_equal(a['w%d' % g], b['w%d' % g])
        assert np.abs(a['theta%d' % g] - b['theta%d' % g]).max() < 2e-6
