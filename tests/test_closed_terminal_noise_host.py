"""CPU (no GPU): action noise on an env whose episodes end early, fused (es_rollout_closedloop_terminal_streams).

* the stream-walk kernel (rollout_closedw_walk.cu) compiles for sm_90a to three depths of tanh and of the other activations,
  none with a stack frame or spills;
* the entry point is declared, bound and built;
* es.step keeps the whole generation on the device for such a policy only with ``BatchedRollout(fuse_noisy_terminal=True)``
  (tanh, and other activations with fuse_activations), and not for the default, MeanRewardResult, binned heads or ac_std = 0;
* the words generated per stream cover what a stream consumes when nothing falls, counted on the CPU with numpy's
  generator at the shapes the GPU tests and the timing tool run."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib, build

NVCC = build.nvcc_path()
HAVE_NVCC = (os.path.isabs(NVCC) and os.path.exists(NVCC)) or shutil.which(NVCC) is not None


@pytest.mark.skipif(not HAVE_NVCC, reason='needs nvcc')
def test_walk_kernels_compile_without_spills():
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c', '-o',
                              os.path.join(tmp, 'w.o'), os.path.join(build.CSRC, 'rollout_closedw_walk.cu')],
                             capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    props = re.findall(r'Function properties for (\S*rollout_closedw_walk_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill '
                       r'stores, (\d+) bytes spill loads', log)
    variants = set()
    for name, stack, st, ld in props:
        assert stack == '0' and st == '0' and ld == '0', f'{name}: {stack} bytes stack, {st} bytes spill stores, {ld} loads'
        m = re.search(r'rollout_closedw_walk_kernelILi(\d)ELb([01])E', name)
        assert m, name
        variants.add((int(m.group(1)), int(m.group(2))))
    assert len(props) == 6 and variants == {(nl, a) for nl in (3, 4, 5) for a in (0, 1)}, log


def test_entry_point_is_declared_bound_and_built():
    with open(os.path.join(build.HERE, '..', 'include', 'es_b200.h')) as f:
        assert 'int es_rollout_closedloop_terminal_streams(' in f.read()
    assert 'es_rollout_closedloop_terminal_streams' in _lib.SIGNATURES
    assert 'rollout_closedw_walk.cu' in build.SOURCES
    # the C signature's parameter count is the binding's
    with open(os.path.join(build.HERE, '..', 'include', 'es_b200.h')) as f:
        decl = re.search(r'int es_rollout_closedloop_terminal_streams\((.*?)\);', f.read(), re.S).group(1)
    assert len(decl.split(',')) == len(_lib.SIGNATURES['es_rollout_closedloop_terminal_streams'][1])


def _policy_and_fit_fn(ac_std=0.01, fall_height=0.5, kind='tanh', binned=False, **kw):
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
    from es_pytorch_b200.nn.nn import FeedForward, FFBinned
    from es_pytorch_b200.nn.optimizers import Adam
    env = ClosedLoopEnv(15, 3, 30, fall_height=fall_height)
    if binned:
        net = FFBinned([32, 32], torch.nn.Tanh(), env, 4)
    else:
        net = FeedForward([32, 32], torch.nn.LeakyReLU(0.1) if kind == 'leaky' else torch.nn.Tanh(), env, ac_std, 5)
    p = Policy(net, 0.05, Adam(len(torch.nn.utils.parameters_to_vector(net.parameters())), 0.01))
    return p, BatchedRollout(env, 30, coins_per_eval=1, **kw)


def _fuses(p, f):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.utils.rankers import CenteredRanker
    return es._can_fuse_step(dist.world(), p, f, CenteredRanker())


def test_the_flag_alone_fuses_a_noisy_generation_whose_episodes_end_early():
    from es_pytorch_b200.gym.training_result import MeanRewardResult
    assert _fuses(*_policy_and_fit_fn(fuse_noisy_terminal=True))
    assert _fuses(*_policy_and_fit_fn(kind='leaky', fuse_noisy_terminal=True, fuse_activations=True))
    assert not _fuses(*_policy_and_fit_fn())                                             # the default: one evaluation per launch
    assert not _fuses(*_policy_and_fit_fn(kind='leaky', fuse_noisy_terminal=True))       # the module's own forward
    assert not _fuses(*_policy_and_fit_fn(fuse_noisy_terminal=True, result=MeanRewardResult))
    # routes the flag does not change: the fused terminal route without noise, and binned heads (which draw none)
    assert _fuses(*_policy_and_fit_fn(ac_std=0.0))
    assert _fuses(*_policy_and_fit_fn(ac_std=0.0, fuse_noisy_terminal=True))
    assert _fuses(*_policy_and_fit_fn(ac_std=0.0, binned=True, fuse_noisy_terminal=True))


HARNESS = r'''
#include <stdarg.h>
#include <stdio.h>
#include "%s"
void es_set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vfprintf(stdout, fmt, ap); va_end(ap); printf("\n"); }
int es_ctx_scratch(es_ctx*, size_t, void**) { return ES_ERR_NOMEM; }
int main(int argc, char** argv) {
    es_ctx ctx = {};
    ctx.sm_count = 132;
    int streams, pairs, coins, N;
    while (scanf("%%d %%d %%d %%d", &streams, &pairs, &coins, &N) == 4) {
        EsStreamWords w;
        const int rc = es_impl_stream_words_plan(&ctx, "plan", streams, pairs, coins, N, &w);
        printf("rc %%d limit %%u need %%lld\n", rc, rc ? 0u : w.limit, mg_blocks_needed(pairs, coins, N));
    }
    return 0;
}
'''


def _accepts(words):
    """numpy's legacy_gauss accept test of the 4-word attempt starting at every word."""
    w = words.astype(np.uint64)
    u = ((w[:-1] >> 5) * 67108864 + (w[1:] >> 6)).astype(np.float64) / 9007199254740992.0       # random_sample of words i, i+1
    x1, x2 = 2.0 * u[:-2] - 1.0, 2.0 * u[2:] - 1.0
    r2 = x1 * x1 + x2 * x2
    return (r2 < 1.0) & (r2 != 0.0)


def _consumed(seed, pairs, coins, N, upper):
    """The words one stream consumes for `pairs` pairs when nothing falls: randint (masked rejection), the coins, N gaussians
    per evaluation (the cache carried over), counted on numpy's own word stream."""
    words = np.random.RandomState(seed).randint(0, 2 ** 32, size=2_000_000, dtype=np.uint32)
    acc = _accepts(words)
    mask = (1 << int(upper - 1).bit_length()) - 1
    cur, cached = 0, 0
    for _ in range(pairs):
        while (int(words[cur]) & mask) > upper - 1:
            cur += 1
        cur += 1
        for _ in range(2):
            cur += 2 * coins
            need = (N - cached + 1) // 2
            hits = np.flatnonzero(acc[cur::4])
            cur += 4 * (hits[need - 1] + 1) if need else 0
            cached = (N - cached) % 2 if need else cached - N
    return cur


@pytest.mark.skipif(not HAVE_NVCC, reason='needs nvcc')
def test_generated_words_cover_the_no_fall_consumption():
    # (the last three: more streams than the fill's 4 segments per SM, where the segment length is capped by the need)
    cases = [(3, 4, 1, 60 * 3), (1, 5, 0, 2 * 60 * 4), (3, 2, 1, 3 * 30 * 8), (8, 30, 1, 1000 * 3), (150, 1, 1, 20 * 3),
             (529, 4, 1, 1000 * 3), (600, 4, 1, 1000 * 3), (2400, 1, 1, 1000 * 3)]
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, 'plan.cu'), os.path.join(tmp, 'plan')
        with open(src, 'w') as f:
            f.write(HARNESS % os.path.join(build.CSRC, 'mt_gauss.cu').replace('\\', '/'))
        res = subprocess.run([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-std=c++17', '-o', exe, src], capture_output=True,
                             text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        out = subprocess.run([exe], input=''.join(f'{s} {n} {c} {N}\n' for s, n, c, N in cases), capture_output=True, text=True,
                             timeout=60).stdout
    plans = [(int(m.group(2)), int(m.group(3))) for m in re.finditer(r'rc (-?\d+) limit (\d+) need (\d+)', out)]
    assert len(plans) == len(cases), out
    for (s, n, c, N), (limit, need) in zip(cases, plans):
        used = max(_consumed(seed, n, c, N, 10 ** 6) for seed in range(4))
        # a stream starts at most 624 words into its block 0 and the walk stages at most 256 words past its cursor
        assert used + 624 + 256 <= limit, (s, n, c, N, used, limit)
        # what is generated stays within twice the mean + 12 sigma bound, whatever the number of streams
        assert limit + 8 <= (2 * need + 1) * 624, (s, n, c, N, limit, need)
        print(f'streams {s} pairs {n} coins {c} gaussians {N}: consumed <= {used} words, bound {need * 624}, generated {limit}')
