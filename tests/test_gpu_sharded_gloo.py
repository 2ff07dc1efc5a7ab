"""The sharded generation on one GPU: W = 2 and W = 3 processes over gloo, against one process holding every rank's stream.

Every feature of the generation is checked elsewhere with world size 1, its ranks as virtual ones in one process.  What only
a world size above 1 runs is how the ranks' work is put together: each process's shard offset (``k_begin``), the one
allgather of the fitness rows, indices and statistics, the sum of the shared statistics row, the allreduce of the partial
gradient, ``approx_grad``'s shard bounds (including the odd ``K`` of an elite ranker, where rank 0 reconstructs everything),
``ObStat.mpi_inc`` and the steps' ``allgather_object``.  Several processes share the one GPU by time-slicing.

This module is also the worker.  The module-scoped fixture runs it twice per W: under ``torch.distributed.run`` with W
processes (gloo), and alone as the one-process reference, which holds all 3 W streams (3 per process in the sharded run).
One launch runs every route below, two generations of es.step each, and writes one ``.npz`` per route; the cases read
those.  The open-loop float32 route adds a third generation through ``DeviceGeneration.run``, whose processes rank only
their own shard of pairs (es.step ranks all K on every process).

Per route and generation, against the one-process run:
  * exact: all K noise indices in rank-major order, the ranked weights, ``n_fits_ranked``, every stream's whole MT19937
    state, the ObStat count and ``steps``;
  * fitness rows bit for bit, except where the rollout kernel a process runs depends on its pair count (``_dispatch``
    restates the float32 launcher's choice, and the case asserts which of the two a route is in): there each run is held to
    test_gpu_rollout_f64.py's per-evaluation float64 bound, and the rows must differ somewhere;
  * ObStat sums: the sharded order sums per process and then across processes, so the two runs agree to
    ``n 2^-53`` of the sum of the terms' magnitudes (bounded by ``sqrt(count * sumsq)``, Cauchy-Schwarz);
  * the allreduced gradient sum against float64 ``sum_k w_k eps_k`` over all K, within ``(K + 1) 2^-24 sum_k |w_k||eps_k|``;
    theta within test_gpu_multi.py's 2e-6 wherever the gradient is resolved (``_assert_theta_close``), and every process's
    theta the same bit for bit.
Generation 1 starts both runs from the same theta (``_Worker.restart``), so that its fitness rows compare bit for bit too.
The collectives take the generation's CUDA tensors as they are: gloo gathers and reduces CUDA tensors itself.
The open-loop float32 route is also held to the oracle (indices, weights, states, theta, and the ObStat against the oracle's
per-process accumulation summed across processes); the one-process runs of
the other routes are checked against the oracle and float64 in the files that own them.
"""
import math
import os
import signal
import socket
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

pytestmark = pytest.mark.gpu

U24, U53 = 2.0 ** -24, 2.0 ** -53
PER_PROC = 3                  # streams (virtual ranks) per process in the sharded run
ROUTES = ('open_f32_adam', 'open_tc3_noise', 'closed_cluster', 'fall_fused', 'fall_mean_reward', 'fall_noisy_per_eval',
          'nsra', 'ns_novelty', 'elite_odd', 'binned_f32', 'relu_tc3', 'opaque_fit_fn')
SM_COUNT_H100 = 132
EVAL_REL_F32 = 1e-5           # test_gpu_rollout_f64.py's per-evaluation bound for ES_ROLLOUT_F32, relative to the reward mass


# ============================================================================================ the worker
class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _theta0(sizes, gain, seed):
    rs = np.random.RandomState(seed)
    return np.concatenate([rs.randn(fi * fo + fo) * (gain / math.sqrt(fi))
                           for fi, fo in zip(sizes[:-1], sizes[1:])]).astype(np.float32)


class _Worker:
    def __init__(self, out_dir, W):
        import torch
        from es_pytorch_b200 import dist
        from es_pytorch_b200.engine import get_engine
        self.torch, self.dist = torch, dist
        self.comm = dist.init_from_env('gloo')
        self.eng = get_engine(0)
        self.out_dir, self.W = out_dir, W
        self.S = PER_PROC * W
        self.per = self.S // self.comm.size
        self.last_gsum = None
        grad_reconstruct = self.eng.grad_reconstruct

        def capture(*a, **kw):                # the partial sum each process reconstructs; the allreduce sums it in place
            out = grad_reconstruct(*a, **kw)
            self.last_gsum = out
            return out
        self.eng.grad_reconstruct = capture

    def mine(self, seq):
        r = self.comm.rank
        return list(seq[self.per * r:self.per * (r + 1)])

    def states(self, streams):
        """Every stream of every process, rank-major: key [S, 624], pos, has_gauss, cached gaussian."""
        local = [s.get_state() for s in streams]
        local = [(np.asarray(st[1], np.uint32), int(st[2]), int(st[3]), float(st[4])) for st in local]
        every = [x for part in self.comm.allgather_object(local) for x in part]
        return (np.stack([x[0] for x in every]), np.array([x[1] for x in every]), np.array([x[2] for x in every]),
                np.array([x[3] for x in every]))

    def save(self, name, rec):
        if self.comm.rank == 0:
            np.savez(os.path.join(self.out_dir, name + '.npz'), **rec)

    # ---------------------------------------------------------------------------------------- building blocks
    def policy(self, net, sizes, gain, seed, std=0.02):
        from es_pytorch_b200.core.policy import Policy
        from es_pytorch_b200.nn.optimizers import Adam
        P = sum(fi * fo + fo for fi, fo in zip(sizes[:-1], sizes[1:]))
        p = Policy(net, std, Adam(P, 0.01))
        p.flat_params[...] = _theta0(sizes, gain, seed)
        p.set_nn_params(p.flat_params)
        return p

    def table(self, P, seed):
        from es_pytorch_b200.core.noisetable import NoiseTable
        t = np.random.RandomState(seed).randn(P + 60_000).astype(np.float32)
        return NoiseTable(P, t), t

    def streams(self, base):
        return [np.random.RandomState(base + 7 * r) for r in range(self.S)]

    def steps_of_es_step(self, name, policy, nt, table, env, make_fit, ranker, n, seeds, gens=2, fused=None, run=False):
        """Two generations of es.step; per generation everything the cases compare.  ``run``: a third generation through
        ``DeviceGeneration.run`` on the generation es.step cached, where every process ranks its own shard of pairs
        (``update(all_weights=False)``, the call bench.py times) instead of all K."""
        from es_pytorch_b200.core import es
        from es_pytorch_b200.utils.reporters import Reporter

        class Rec(Reporter):
            def log_gen(self, fits, noiseless_tr, policy, steps):
                self.steps = steps
        streams = self.mine(self.streams(seeds))
        fit_fn = make_fit(streams)
        if fused is not None:
            assert es._can_fuse_step(self.comm, policy, fit_fn, ranker) == fused, name
        cfg = _Cfg(general=_Cfg(policies_per_gen=2 * n * self.comm.size, batch_size=500), policy=_Cfg(l2coeff=0.005))
        rec = dict(table=table, n=n, K=n * self.S, sigma=policy.std)
        for g in range(gens):
            self.restart(policy, g, rec)
            rec['theta_in%d' % g] = policy.flat_params.copy()
            self.last_gsum = None
            rep = Rec()
            _, ob = es.step(cfg, self.comm, policy, nt, env, fit_fn, streams[0], ranker, rep)
            self._record(rec, g, ranker, policy, ob, rep.steps, streams)
        if run:
            self._run_generation(rec, gens, policy, fit_fn._gen, n)
        rec['gens'] = gens + bool(run)
        self.save(name, rec)

    def _run_generation(self, rec, g, policy, gen, n):
        """Generation g through gen.run(n): the shard-local rank call, reconstruction, allreduce and optimizer step."""
        self.restart(policy, g, rec)
        rec['theta_in%d' % g] = policy.flat_params.copy()
        policy.theta_dev(gen.eng)                           # the new theta into the generation's device theta
        gen.l2coeff, gen.ranker = 0.005, None               # es.step leaves l2coeff at 0: approx_grad passes its own
        gen.run(n)
        gen.eng.sync()
        multi = self.comm.size > 1
        assert gen.weights.numel() == gen.k_local and (gen.weights_all is None) == multi     # this process's shard was ranked
        rec['inds%d' % g] = (gen.idx_all if multi else gen.idx).cpu().numpy().astype(np.float64)
        rec['w%d' % g] = np.concatenate(self.comm.allgather_object(gen.weights.cpu().numpy())).astype(np.float64)
        rec['n_ranked%d' % g] = 2 * gen.K
        rec['pos%d' % g] = (gen.fpos_all if multi else gen.fit_local[0]).cpu().numpy()
        rec['neg%d' % g] = (gen.fneg_all if multi else gen.fit_local[1]).cpu().numpy()
        theta = gen.theta.cpu().numpy()
        rec['theta%d' % g] = theta
        rec['theta_ranks%d' % g] = np.stack(self.comm.allgather_object(theta))
        rec['gsum%d' % g] = gen.gsum.cpu().numpy()
        st, d = gen._gen_stats.cpu().numpy(), gen.obs_dim
        rec['ob_sum%d' % g], rec['ob_sumsq%d' % g], rec['ob_count%d' % g] = st[:d], st[d:2 * d], st[2 * d]
        rec['key%d' % g], rec['mtpos%d' % g], rec['has%d' % g], rec['gauss%d' % g] = self.states(gen.rank_states())

    @staticmethod
    def restart(policy, g, rec):
        """Generation g > 0 starts from a theta of its own, written into flat_params as a script may write it.  After a
        generation the thetas of the two runs differ in their last bits (the gradient was summed in another order), and
        from the same theta the next generation's fitness rows can be compared bit for bit again.  The streams, the
        optimizer's moments and the cached device generation carry over."""
        if g:
            step = np.random.RandomState(77 + g).randn(len(policy)).astype(np.float32) * np.float32(1e-3)
            policy.flat_params[...] = rec['theta_in0'] + step
            policy.set_nn_params(policy.flat_params)

    def _record(self, rec, g, ranker, policy, ob, steps, streams):
        rec['inds%d' % g] = np.asarray(ranker.noise_inds, dtype=np.float64)
        rec['w%d' % g] = np.asarray(ranker.ranked_fits, dtype=np.float64).reshape(-1)
        rec['n_ranked%d' % g] = ranker.n_fits_ranked
        rec['pos%d' % g] = np.asarray(ranker.fits_pos, dtype=np.float64)
        rec['neg%d' % g] = np.asarray(ranker.fits_neg, dtype=np.float64)
        rec['theta%d' % g] = policy.flat_params.copy()
        rec['theta_ranks%d' % g] = np.stack(self.comm.allgather_object(policy.flat_params.copy()))
        rec['gsum%d' % g] = self.last_gsum.cpu().numpy()
        rec['ob_sum%d' % g], rec['ob_sumsq%d' % g], rec['ob_count%d' % g] = ob.sum.copy(), ob.sumsq.copy(), ob.count
        rec['steps%d' % g] = steps
        rec['key%d' % g], rec['mtpos%d' % g], rec['has%d' % g], rec['gauss%d' % g] = self.states(streams)

    # ---------------------------------------------------------------------------------------- the routes
    def open_loop(self, name, sizes, T, n, mode, gain=1.0, ac_std=0.0, episodes=1, activation=None, fuse=False,
                  result=None, archive=None, ranker=None, fused=True, run=False, seeds=1000):
        import torch
        from es_pytorch_b200.gym.batched import BatchedRollout
        from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
        from es_pytorch_b200.nn.nn import FeedForward
        from es_pytorch_b200.utils.rankers import CenteredRanker
        env = SyntheticEnv(sizes[0], sizes[-1], T)
        net = FeedForward(list(sizes[1:-1]), activation or torch.nn.Tanh(), env, ac_std, 5)
        policy = self.policy(net, sizes, gain, seeds + 1)
        nt, table = self.table(len(policy), seeds + 2)
        kw = dict(coins_per_eval=1, save_obs_chance=0.2, rollout_mode=mode, episodes=episodes, fuse_activations=fuse)
        if result is not None:
            kw['result'] = result
        if archive is not None:
            kw['archive'] = archive
        self.steps_of_es_step(name, policy, nt, table, env, lambda st: BatchedRollout(env, T, rank_streams=st, **kw),
                              ranker or CenteredRanker(), n, seeds, fused=fused, run=run)

    def closed_loop(self, name, sizes, T, n, gain=1.0, fall_height=None, ac_std=0.0, result=None, fused=True, seeds=2000):
        import torch
        from es_pytorch_b200.gym.batched import BatchedRollout
        from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
        from es_pytorch_b200.nn.nn import FeedForward
        from es_pytorch_b200.utils.rankers import CenteredRanker
        env = ClosedLoopEnv(sizes[0], sizes[-1], T, fall_height=fall_height)
        net = FeedForward(list(sizes[1:-1]), torch.nn.Tanh(), env, ac_std, 5)
        policy = self.policy(net, sizes, gain, seeds + 1, std=0.05)
        nt, table = self.table(len(policy), seeds + 2)
        kw = dict(coins_per_eval=1, save_obs_chance=0.2)
        if result is not None:
            kw['result'] = result
        self.steps_of_es_step(name, policy, nt, table, env, lambda st: BatchedRollout(env, T, rank_streams=st, **kw),
                              CenteredRanker(), n, seeds, fused=fused)

    def binned(self, name, T, n, seeds=3000):
        import torch
        from es_pytorch_b200 import _lib
        from es_pytorch_b200.gym.batched import BatchedRollout
        from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
        from es_pytorch_b200.nn.nn import FFBinned
        from es_pytorch_b200.utils.rankers import CenteredRanker
        env = SyntheticEnv(17, 6, T)
        net = FFBinned([32, 32], torch.nn.Tanh(), env, 5)
        policy = self.policy(net, [17, 32, 32, 30], 1.0, seeds + 1)
        nt, table = self.table(len(policy), seeds + 2)
        self.steps_of_es_step(name, policy, nt, table, env,
                              lambda st: BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.2, rank_streams=st,
                                                        rollout_mode=_lib.ES_ROLLOUT_F32),
                              CenteredRanker(), n, seeds, fused=True)

    def opaque(self, name, T, n, seeds=4000):
        """An opaque python fit_fn (the scripts' rs.random() coin and run_model): es.test_params call by call, then
        Ranker.rank and approx_grad.  One stream per process, as a script has; the one-process reference runs test_params
        once per virtual rank and joins the rows, statistics and steps in rank order, as the collectives do."""
        import torch
        from es_pytorch_b200.core import es
        from es_pytorch_b200.gym.gym_runner import run_model
        from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
        from es_pytorch_b200.gym.training_result import RewardResult
        from es_pytorch_b200.nn.nn import FeedForward
        from es_pytorch_b200.nn.obstat import ObStat
        from es_pytorch_b200.utils.rankers import CenteredRanker
        sizes = [17, 32, 32, 6]
        env = SyntheticEnv(17, 6, T)
        policy = self.policy(FeedForward([32, 32], torch.nn.Tanh(), env, 0.0, 5), sizes, 1.0, seeds + 1)
        nt, table = self.table(len(policy), seeds + 2)
        all_streams = [np.random.RandomState(seeds + 7 * r) for r in range(self.W)]
        ranks = [self.comm.rank] if self.comm.size > 1 else list(range(self.W))

        def fit_fn(rs):
            def fit(model, use_ac_noise=True):
                save = rs.random() < 0.2
                rews, behv, obs, steps = run_model(model, env, T, rs if use_ac_noise else None)
                return RewardResult(rews, behv, obs if save else np.array([np.zeros(env.observation_space.shape)]), steps)
            return fit
        rec = dict(table=table, n=n, K=n * self.W, sigma=policy.std, gens=2)
        ranker = CenteredRanker()
        for g in range(2):
            self.restart(policy, g, rec)
            rec['theta_in%d' % g] = policy.flat_params.copy()
            parts, ob, steps = [], ObStat(env.observation_space.shape, 0), 0
            for r in ranks:
                part_ob = ObStat(env.observation_space.shape, 0)
                pos, neg, inds, st = es.test_params(self.comm, n, policy, nt, part_ob, fit_fn(all_streams[r]), all_streams[r])
                parts.append((pos, neg, inds))
                ob.inc(part_ob.sum, part_ob.sumsq, part_ob.count)
                steps += st
            pos, neg, inds = (np.concatenate([p[i] for p in parts]) for i in range(3))
            ranker.rank(pos, neg, inds)
            self.last_gsum = None
            es.approx_grad(policy, ranker, nt, policy.flat_params, 500, 0.005)
            self._record(rec, g, ranker, policy, ob, steps, [all_streams[r] for r in ranks])
        self.save(name, rec)

    def noise_table(self):
        """NoiseTable.create_shared: rank 0 picks the seed, every process draws its replica on the device."""
        from es_pytorch_b200.core.noisetable import NoiseTable
        torch, comm, eng = self.torch, self.comm, self.eng

        class SeedReporter:
            seed = None

            def print(self, s):
                if s.startswith('nt seed:'):
                    self.seed = int(s.split(':')[1])
        rep = SeedReporter()
        size = 1_000_003
        nt = NoiseTable.create_shared(comm, size, 1000, rep)
        t = nt.device_table(eng)
        check = torch.stack([t.double().sum(), t.view(torch.int32).to(torch.int64).sum().double()])
        checks = torch.empty(comm.size, 2, dtype=torch.float64, device=eng.device)
        comm.allgather_into(checks, check)
        offs = torch.from_numpy(np.random.RandomState(9).randint(0, size - 32, 1000)).to(eng.device)
        sl = t[offs[:, None] + torch.arange(32, device=eng.device)[None, :]]
        slices = torch.empty(comm.size, 1000, 32, dtype=torch.float32, device=eng.device)
        comm.allgather_into(slices, sl)
        self.save('noise_table', dict(seed=rep.seed if rep.seed is not None else -1, size=size, offs=offs.cpu().numpy(),
                                      checks=checks.cpu().numpy(), slices=slices.cpu().numpy()))

    def run(self):
        import torch
        from es_pytorch_b200 import _lib
        from es_pytorch_b200.gym.training_result import MeanRewardResult, NSResult
        from es_pytorch_b200.utils.rankers import CenteredRanker, EliteRanker, MultiObjectiveRanker
        F32, TC3 = _lib.ES_ROLLOUT_F32, _lib.ES_ROLLOUT_TC3
        wide = [15, 256, 256, 3]
        archive = np.random.RandomState(21).randn(12, 2) * 0.05
        self.open_loop('open_f32_adam', [376, 64, 64, 17], 32, 8, F32, gain=1.0, run=True, seeds=1000)
        self.open_loop('open_tc3_noise', wide, 40, 4, TC3, ac_std=0.01, episodes=2, seeds=1100)
        self.closed_loop('closed_cluster', wide, 40, 4, seeds=2000)
        # 15-32-32-3 at gain 1.5 and h = 0.5: some evaluations fall, none at step 0 (test_gpu_closed_terminal.py's setup)
        fall = dict(sizes=[15, 32, 32, 3], T=60, n=4, gain=1.5, fall_height=0.5)
        self.closed_loop('fall_fused', seeds=2100, **fall)
        self.closed_loop('fall_mean_reward', result=MeanRewardResult, fused=False, seeds=2200, **fall)
        self.closed_loop('fall_noisy_per_eval', ac_std=0.01, fused=False, seeds=2300, **fall)
        self.open_loop('nsra', wide, 40, 4, TC3, archive=archive, ranker=MultiObjectiveRanker(CenteredRanker(), 0.5),
                       seeds=1200)
        self.open_loop('ns_novelty', wide, 40, 4, TC3, archive=archive, result=NSResult, seeds=1300)
        # 2K fitnesses, elite count 7: odd, and divides over neither 2 nor 3 processes
        K = 4 * self.S
        self.open_loop('elite_odd', [17, 32, 32, 6], 32, 4, F32, ranker=EliteRanker(CenteredRanker(), 7.5 / (2 * K)),
                       fused=False, seeds=1400)
        self.binned('binned_f32', 32, 4)
        self.open_loop('relu_tc3', wide, 40, 4, TC3, activation=torch.nn.ReLU(), fuse=True, seeds=1500)
        self.opaque('opaque_fit_fn', 20, 4)
        self.noise_table()
        self.comm.barrier()
        os.write(1, ('SHARDED_OK_%d\n' % self.comm.rank).encode())


# ============================================================================================ the launches
def _free_port():
    with socket.socket() as sk:
        sk.bind(('127.0.0.1', 0))
        return sk.getsockname()[1]


def _launch(cmd, timeout):
    """Runs ``cmd`` in a session of its own; on a timeout the whole process group is killed, so no worker outlives it."""
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=ROOT,
                            start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        out, _ = proc.communicate()
        raise AssertionError(f'{cmd[-3:]} did not finish in {timeout} s; its process group was killed\n{out[-3000:]}')
    assert proc.returncode == 0, out[-4000:]
    return out


@pytest.fixture(scope='module', params=[2, 3], ids=['W2', 'W3'])
def runs(request, tmp_path_factory):
    W = request.param
    one, shard = tmp_path_factory.mktemp(f'one{W}'), tmp_path_factory.mktemp(f'shard{W}')
    me = os.path.abspath(__file__)
    out = _launch([sys.executable, me, str(one), str(W)], timeout=150)
    assert 'SHARDED_OK_0' in out
    out = _launch([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={W}', '--master-addr',
                   '127.0.0.1', '--master-port', str(_free_port()), me, str(shard), str(W)], timeout=200)
    assert all(f'SHARDED_OK_{r}' in out for r in range(W)), out[-3000:]
    return W, one, shard


# ============================================================================================ the checks
def _dispatch(sizes, T, pairs, sm=SM_COUNT_H100):
    """rollout_f32.cu's es_impl_rollout_f32 for a tanh MLP: ('packed', 1) for the packed-FMA kernel, else ('general',
    the time splits of the episode) -- both depend on the launch's pair count.  test_gpu_rollout_f64.py's _uses_f32x."""
    from test_gpu_rollout_f64 import _uses_f32x
    if _uses_f32x(sizes, pairs, sm):
        return 'packed', 1
    n_tiles = -(-T // 32)
    splits = min(max(sm // (2 * pairs), 1), n_tiles) if 2 * pairs < sm else 1
    return 'general', splits


# the float32 routes whose rollout kernel could depend on the pair count: (layer sizes, T); every other route's kernel
# evaluates each pair alike whatever the launch's pair count (tensor-core and cluster kernels; binned and the episode
# length of one time tile for the general float32 kernel)
F32_ROUTES = {'open_f32_adam': ([376, 64, 64, 17], 32), 'elite_odd': ([17, 32, 32, 6], 32), 'binned_f32': ([17, 32, 32, 30], 32)}


def _bitwise_route(route, W, n):
    if route not in F32_ROUTES:
        return True
    sizes, T = F32_ROUTES[route]
    if route == 'binned_f32':                            # binned heads always run the general kernel
        return True
    return _dispatch(sizes, T, n * PER_PROC) == _dispatch(sizes, T, n * PER_PROC * W)


def _load(d, route):
    return dict(np.load(os.path.join(d, route + '.npz')))


def _f64_fitness_bound(a, route, g):
    """Each evaluation of ``a``'s generation ``g`` within EVAL_REL_F32 of the float64 truth's reward mass."""
    import f64_rollout as f64
    from oracle import es_oracle as orc
    sizes, T = F32_ROUTES[route]
    spec = orc.SyntheticEnvSpec(sizes[0], sizes[-1], T)
    obsn = orc.normalise_obs(spec.obs_stream[:T], np.zeros(sizes[0]), np.ones(sizes[0]), 5.0)
    tf, _, mass, _ = f64.rollout_f64(a['table'], a['inds%d' % g].astype(np.int64), a['theta_in%d' % g], float(a['sigma']),
                                     sizes, obsn, spec.rew_vec[:T], spec.pos_scale)
    got = np.stack([a['pos%d' % g].reshape(-1), a['neg%d' % g].reshape(-1)])
    err = np.abs(got - tf)
    assert np.all(err <= EVAL_REL_F32 * mass), (route, g, float((err / mass).max()))


def _gsum_truth(a, g):
    table, w = a['table'].astype(np.float64), a['w%d' % g]
    inds = a['inds%d' % g].astype(np.int64)
    P = a['gsum%d' % g].size
    eps = np.stack([table[i:i + P] for i in inds])
    return w @ eps, np.abs(w) @ np.abs(eps)


def _assert_theta_close(a, theta, g, tag, l2coeff=0.005, lr=0.01):
    """``theta`` (another run's, or the oracle's) against run ``a``'s after generation g: within test_gpu_multi.py's 2e-6
    wherever the optimizer's input h = l2coeff theta - gsum / n_fits_ranked is resolved.  Adam moves an element by about
    lr h / (|h| + 1e-8), so where h is within its float32 rounding of 0 (the gradient sum cancels), or near Adam's
    epsilon, any step of at most lr is as right as another: there theta is held to 2 lr, and such elements must be few."""
    truth, absum = _gsum_truth(a, g)
    n_ranked, nk = float(a['n_ranked%d' % g]), a['inds%d' % g].size
    th = a['theta_in%d' % g].astype(np.float64)
    h = l2coeff * th - truth / n_ranked
    dh = (nk + 1) * U24 * absum / n_ranked + 4 * U24 * l2coeff * np.abs(th)
    ok = np.abs(h) >= np.maximum(256 * dh, 1e-6)
    d = np.abs(a['theta%d' % g].astype(np.float64) - theta)
    assert ok.mean() >= 0.99, f'{tag}: only {ok.mean():.3f} of the gradient is resolved'
    assert d[ok].max() < 2e-6, f'{tag}: theta, {d[ok].max():.3g} where the gradient is resolved'
    assert d.max() <= 2 * lr, f'{tag}: theta, {d.max():.3g}'


@pytest.mark.parametrize('route', ROUTES)
def test_sharded_generation_matches_one_process(runs, route):
    W, one_dir, shard_dir = runs
    a, b = _load(one_dir, route), _load(shard_dir, route)
    n, K = int(a['n']), int(a['K'])
    assert int(b['K']) == K and np.array_equal(a['table'], b['table'])
    bitwise = _bitwise_route(route, W, n)
    # which case a route is in: only the open-loop float32 shape at W = 3 straddles the packed-FMA dispatch
    assert bitwise == (route != 'open_f32_adam' or W == 2), (route, W, 'dispatch changed: review _dispatch and F32_ROUTES')
    gens = int(a['gens'])
    assert gens == int(b['gens']) == (3 if route == 'open_f32_adam' else 2)
    for g in range(gens):
        tag = f'{route} W={W} generation {g}'
        # the exact quantities
        n_inds = int(a['n_ranked%d' % g]) if route == 'elite_odd' else K      # the elite's indices, else all K
        assert a['inds%d' % g].size == n_inds and np.array_equal(a['inds%d' % g], b['inds%d' % g]), f'{tag}: noise indices'
        assert np.array_equal(a['w%d' % g], b['w%d' % g]), f'{tag}: ranked weights'
        assert int(a['n_ranked%d' % g]) == int(b['n_ranked%d' % g]), f'{tag}: n_fits_ranked'
        for k in ('key', 'mtpos', 'has', 'gauss'):
            assert np.array_equal(a[k + '%d' % g], b[k + '%d' % g]), f'{tag}: stream {k}'
        assert float(a['ob_count%d' % g]) == float(b['ob_count%d' % g]), f'{tag}: ObStat count'
        if 'steps%d' % g in a:                             # es.step's (DeviceGeneration.run reports none)
            assert int(a['steps%d' % g]) == int(b['steps%d' % g]), f'{tag}: steps'
        # fitness rows
        fa = np.stack([a['pos%d' % g], a['neg%d' % g]])
        fb = np.stack([b['pos%d' % g], b['neg%d' % g]])
        if bitwise:
            assert np.array_equal(fa.view(np.int64), fb.view(np.int64)), f'{tag}: fitness rows'
        else:
            assert not np.array_equal(fa, fb), f'{tag}: the two dispatches gave identical rows'
            _f64_fitness_bound(a, route, g)
            _f64_fitness_bound(b, route, g)
        # ObStat sums: per-process sums, then the cross-process sum
        cnt = float(a['ob_count%d' % g])
        n_terms = cnt + W
        mag = np.sqrt(cnt * a['ob_sumsq%d' % g])
        assert np.all(np.abs(a['ob_sum%d' % g] - b['ob_sum%d' % g]) <= n_terms * U53 * mag), f'{tag}: ObStat sum'
        assert np.all(np.abs(a['ob_sumsq%d' % g] - b['ob_sumsq%d' % g]) <= n_terms * U53 * a['ob_sumsq%d' % g]), \
            f'{tag}: ObStat sumsq'
        # the allreduced gradient sum, every run against float64
        for run, x in (('one process', a), ('sharded', b)):
            truth, absum = _gsum_truth(x, g)
            nk = x['inds%d' % g].size
            err = np.abs(x['gsum%d' % g].astype(np.float64) - truth)
            assert np.all(err <= (nk + 1) * U24 * absum), f'{tag}: {run} gradient sum, {float((err / absum).max()):.3g}'
        _assert_theta_close(a, b['theta%d' % g], g, tag)
        # every process steps the same theta: the replicated optimizer on the one allreduced gradient
        th = b['theta_ranks%d' % g]
        assert th.shape[0] == W and all(np.array_equal(th[r], th[0]) for r in range(th.shape[0])), f'{tag}: theta differs between processes'
    # the routes are not vacuous
    assert float(a['ob_count1']) > 0, f'{route}: no observation was saved'
    if route.startswith('fall'):
        T = 60
        steps = int(a['steps0'])
        assert 0 < steps < 2 * K * (T - 1), f'{route}: no evaluation fell ({steps} steps)'
    if route == 'elite_odd':
        nr = int(a['n_ranked0'])
        assert nr == 7 and nr % W != 0


def _obstat_per_process(states, table_len, P, n, W, obs_rows, chance):
    """The oracle's ObStat of one open-loop generation as the processes form it, from copies of the streams: each process
    accumulates its own streams' evaluations in order (stream, pair, + then -; es.py:67-74 and obstat.py:19-22), and the
    W partial records are then summed.  Returns the partials [(sum, sumsq, count)] in rank order."""
    from oracle import es_oracle as orc
    s, q, c = orc.ob_sum_sq_cnt(obs_rows)
    zeros = np.zeros_like(s)
    parts = []
    for r in range(W):
        st = orc.ObStatOracle(s.shape, 0)
        for state in states[PER_PROC * r:PER_PROC * (r + 1)]:
            rs = np.random.RandomState()
            rs.set_state(state.get_state())
            for _ in range(n):
                orc.sample_idx(table_len, rs, P)
                for _sign in range(2):
                    if rs.random() < chance:
                        st.inc(s, q, c)
                    else:
                        st.inc(zeros, zeros, 0)
        parts.append((st.sum, st.sumsq, st.count))
    return parts


def _assert_obstat_is_the_per_process_restatement(b, g, parts, tag):
    """The sharded ObStat against the partial records summed: exact count; the sums within (W - 1) 2^-53 of the partials'
    magnitudes, the rounding of a sum of W float64 records in whatever order the cross-process sum takes."""
    W = len(parts)
    for i, key in enumerate(('ob_sum', 'ob_sumsq')):
        want = sum(p[i] for p in parts)
        mag = sum(np.abs(p[i]) for p in parts)
        err = np.abs(b['%s%d' % (key, g)] - want)
        assert np.all(err <= (W - 1) * U53 * mag), f'{tag}: {key} against the per-process restatement'
    assert float(b['ob_count%d' % g]) == float(sum(p[2] for p in parts)), f'{tag}: ObStat count'


def test_open_loop_f32_route_is_the_oracles_es_step(runs):
    """The sharded open-loop float32 route against the oracle over all 3 W streams: two generations of es.step, then one of
    DeviceGeneration.run (the oracle's generation, with no noiseless evaluation).  Indices, weights and n_fits_ranked
    exact, every stream's state exact, ObStat against the oracle's per-process restatement, theta within 2e-6."""
    from oracle import es_oracle as orc
    W, _, shard_dir = runs
    b = _load(shard_dir, 'open_f32_adam')
    sizes, T = F32_ROUTES['open_f32_adam']
    dims = orc.layer_dims(sizes[0], sizes[1:-1], sizes[-1])
    P = orc.n_params(dims)
    flat, opt = b['theta_in0'].copy(), orc.AdamOracle(P, 0.01)
    S, n = PER_PROC * W, int(b['n'])
    states = [np.random.RandomState(1000 + 7 * r) for r in range(S)]
    spec = orc.SyntheticEnvSpec(sizes[0], sizes[-1], T)
    args = (np.zeros(sizes[0]), np.ones(sizes[0]), 5.0, T, 500, 0.005)
    assert int(b['gens']) == 3
    for g in range(3):
        tag = f'oracle W={W} generation {g}'
        flat[...] = b['theta_in%d' % g]
        parts = _obstat_per_process(states, len(b['table']), P, n, W, spec.obs_stream[1:T + 1], 0.2)
        if g < 2:
            ref = orc.es_step(b['table'], flat, opt, float(b['sigma']), dims, spec, states, n, *args, coins_per_eval=1,
                              save_obs_chance=0.2)
        else:
            ref = orc.generation(b['table'], flat, opt, float(b['sigma']), dims, spec, [None] * S, n, *args,
                                 coins_per_eval=1, rank_states=states, save_obs_chance=0.2)
        assert np.array_equal(b['inds%d' % g], np.asarray(ref['inds'], np.float64)), tag
        assert np.array_equal(b['w%d' % g], np.asarray(ref['weights'], np.float64)), tag
        assert int(b['n_ranked%d' % g]) == ref['n_ranked'], tag
        assert np.array_equal(b['key%d' % g], np.stack([s.get_state()[1] for s in states])), tag
        assert np.array_equal(b['mtpos%d' % g], [s.get_state()[2] for s in states]), tag
        assert float(ref['obstat'].count) == float(sum(p[2] for p in parts)) > 0, tag
        _assert_obstat_is_the_per_process_restatement(b, g, parts, tag)
        _assert_theta_close(b, flat, g, tag)


def test_shared_noise_table_is_one_table_on_every_process(runs):
    """NoiseTable.create_shared: rank 0's seed reaches every process, and every device replica is the same table --
    checksums and 1 000 sampled slices allgathered -- and numpy's RandomState(seed).randn within one float32 ulp."""
    from es_pytorch_b200.core.noisetable import NoiseTable
    W, _, shard_dir = runs
    d = _load(shard_dir, 'noise_table')
    checks, slices = d['checks'], d['slices']
    assert checks.shape == (W, 2) and slices.shape == (W, 1000, 32)
    for r in range(1, W):
        assert np.array_equal(checks[r], checks[0]), r
        assert np.array_equal(slices[r].view(np.int32), slices[0].view(np.int32)), r
    seed = int(d['seed'])
    assert seed >= 0
    host = NoiseTable.make_noise(int(d['size']), seed)
    want = host[d['offs'][:, None] + np.arange(32)[None, :]]
    ulp = np.spacing(np.abs(want))
    assert np.all(np.abs(slices[0] - want) <= ulp)


if __name__ == '__main__':
    _Worker(sys.argv[1], int(sys.argv[2])).run()
