"""The fused noisy route on an env whose episodes end early (``BatchedRollout(fuse_noisy_terminal=True)``,
es_rollout_closedloop_terminal_streams) sharded over two processes (gloo, sharing one GPU), against one process holding every
stream, with test_gpu_sharded_gloo.py's worker, launches and checks.

What only a world size above 1 runs on this route: each process walks its own streams, the fitness rows, indices, ObStat
and the steps' sum travel in the one allgather, every process ranks all K, the partial gradients are allreduced, and each
process stores its own streams back.  Two generations of es.step; per generation, against the one-process run: all K
indices, the ranked weights, ``n_fits_ranked``, every stream's whole MT19937 state (the cached gaussian included: both runs
draw it with the same kernel), the ObStat count, ``steps`` and the fitness rows bit for bit; the ObStat sums within
``n 2^-53`` of their terms' magnitude; theta as test_gpu_sharded_gloo.py holds it, and the same on every process.

This module is also the worker (``_NoisyWorker``, a test_gpu_sharded_gloo._Worker that runs this one route)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from test_gpu_sharded_gloo import U53, _Worker, _assert_theta_close, _free_port, _launch, _load  # noqa: E402

pytestmark = pytest.mark.gpu

ROUTE, T = 'fall_noisy_fused', 60


class _NoisyWorker(_Worker):
    def run(self):
        import torch
        from es_pytorch_b200.gym.batched import BatchedRollout
        from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
        from es_pytorch_b200.nn.nn import FeedForward
        from es_pytorch_b200.utils.rankers import CenteredRanker
        sizes, seeds = [15, 32, 32, 3], 2400
        env = ClosedLoopEnv(sizes[0], sizes[-1], T, fall_height=0.5)
        net = FeedForward(sizes[1:-1], torch.nn.Tanh(), env, 0.01, 5)
        policy = self.policy(net, sizes, 1.5, seeds + 1, std=0.05)
        nt, table = self.table(len(policy), seeds + 2)
        make = lambda st: BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.2, rank_streams=st, fuse_noisy_terminal=True)
        self.steps_of_es_step(ROUTE, policy, nt, table, env, make, CenteredRanker(), 4, seeds, fused=True)
        self.comm.barrier()
        os.write(1, ('SHARDED_OK_%d\n' % self.comm.rank).encode())


@pytest.fixture(scope='module')
def runs(tmp_path_factory):
    W = 2
    one, shard = tmp_path_factory.mktemp('one'), tmp_path_factory.mktemp('shard')
    me = os.path.abspath(__file__)
    out = _launch([sys.executable, me, str(one), str(W)], timeout=150)
    assert 'SHARDED_OK_0' in out
    out = _launch([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={W}', '--master-addr',
                   '127.0.0.1', '--master-port', str(_free_port()), me, str(shard), str(W)], timeout=200)
    assert all(f'SHARDED_OK_{r}' in out for r in range(W)), out[-3000:]
    return W, one, shard


def test_two_processes_match_one_process(runs):
    W, one_dir, shard_dir = runs
    a, b = _load(one_dir, ROUTE), _load(shard_dir, ROUTE)
    K = int(a['K'])
    assert int(b['K']) == K and int(a['gens']) == int(b['gens']) == 2
    for g in range(2):
        tag = f'W={W} generation {g}'
        assert a['inds%d' % g].size == K and np.array_equal(a['inds%d' % g], b['inds%d' % g]), f'{tag}: noise indices'
        assert np.array_equal(a['w%d' % g], b['w%d' % g]), f'{tag}: ranked weights'
        assert int(a['n_ranked%d' % g]) == int(b['n_ranked%d' % g]), f'{tag}: n_fits_ranked'
        for k in ('key', 'mtpos', 'has', 'gauss'):
            assert np.array_equal(a[k + '%d' % g], b[k + '%d' % g]), f'{tag}: stream {k}'
        assert float(a['ob_count%d' % g]) == float(b['ob_count%d' % g]), f'{tag}: ObStat count'
        assert int(a['steps%d' % g]) == int(b['steps%d' % g]), f'{tag}: steps'
        fa = np.stack([a['pos%d' % g], a['neg%d' % g]])
        fb = np.stack([b['pos%d' % g], b['neg%d' % g]])
        assert np.array_equal(fa.view(np.int64), fb.view(np.int64)), f'{tag}: fitness rows'
        cnt = float(a['ob_count%d' % g])
        mag = np.sqrt(cnt * a['ob_sumsq%d' % g])
        assert np.all(np.abs(a['ob_sum%d' % g] - b['ob_sum%d' % g]) <= (cnt + W) * U53 * mag), f'{tag}: ObStat sum'
        assert np.all(np.abs(a['ob_sumsq%d' % g] - b['ob_sumsq%d' % g]) <= (cnt + W) * U53 * a['ob_sumsq%d' % g]), \
            f'{tag}: ObStat sumsq'
        _assert_theta_close(a, b['theta%d' % g], g, tag)
        th = b['theta_ranks%d' % g]
        assert th.shape[0] == W and all(np.array_equal(th[r], th[0]) for r in range(W)), f'{tag}: theta differs between processes'
    # not vacuous: observations were saved, evaluations fell after their first step, and the streams moved
    assert float(a['ob_count1']) > 0
    steps = int(a['steps0'])
    assert 0 < steps < 2 * K * (T - 1), f'no evaluation fell ({steps} steps)'
    assert np.any(a['has0'] != a['has1']) or np.any(a['mtpos0'] != a['mtpos1'])


if __name__ == '__main__':
    _NoisyWorker(sys.argv[1], int(sys.argv[2])).run()
