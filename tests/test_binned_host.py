"""CPU (no GPU): binned-action policies (FFBinned, src/nn/nn.py:99-117) -- the oracle's action arithmetic against
FFBinned.forward, the head descriptor and the fuse decision, the binned C entry points, and their kernels' ptxas reports."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (low, high) pairs per action dimension: symmetric, shifted, narrow, negative, and widths that are not powers of two
BOUNDS = [(-1.0, 1.0), (-0.3, 2.7), (0.1, 0.35), (-5.5, -1.25), (-1e-3, 7.0), (-0.7, 0.3)]


def _binned_net(bins, low, high, obs=4, hidden=(8,)):
    from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
    from es_pytorch_b200.nn.nn import FFBinned
    env = SyntheticEnv(obs, len(low), 4)
    env.action_space.low = np.asarray(low, dtype=np.float32)
    env.action_space.high = np.asarray(high, dtype=np.float32)
    return FFBinned(list(hidden), torch.nn.Tanh(), env, bins)


def test_oracle_action_is_ffbinned_forward_bit_for_bit():
    """For bins 2..32 and every idx: a network whose last layer is 0 with one larger bias per dimension picks that bin in
    FFBinned.forward; the oracle's float32 sequence gives the same action bits."""
    low = np.array([b[0] for b in BOUNDS], dtype=np.float32)
    high = np.array([b[1] for b in BOUNDS], dtype=np.float32)
    adim = len(BOUNDS)
    ob = torch.from_numpy(np.random.RandomState(0).randn(4).astype(np.float32))
    for bins in range(2, 33):
        net = _binned_net(bins, low, high)
        last = net.model[-2]
        for idx in range(bins):
            with torch.no_grad():
                last.weight.zero_()
                b = torch.zeros(adim, bins)
                b[:, idx] = 0.5
                b[np.arange(adim), (idx + np.arange(adim)) % bins] = 0.5        # one dimension per shifted idx too
                last.bias.copy_(b.reshape(-1))
                got = net(ob, rs=None).numpy()
                raw = net.model(ob).numpy()
            want = orc.binned_action(raw, bins, low, high)
            assert got.dtype == np.float32
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (bins, idx, got, want)


def test_oracle_action_ties_pick_the_first_bin():
    low, high = np.array([-0.3], np.float32), np.array([2.7], np.float32)
    for bins in (2, 5, 11):
        assert orc.binned_action(np.full(bins, 0.25, np.float32), bins, low, high)[0] == low[0]
        out = np.full(bins, 0.25, np.float32)
        out[bins - 1] = 0.5
        out[1] = 0.5
        assert orc.binned_action(out, bins, low, high)[0] == orc.binned_action(np.eye(bins, dtype=np.float32)[1], bins, low,
                                                                               high)[0]


def test_head_descriptor_and_fuse_decision():
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    from es_pytorch_b200.nn.nn import BinnedHead, FeedForward, FFBinned, FFIntegGausAction
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker, EliteRanker
    env = SyntheticEnv(15, 3, 20)
    net = FFBinned([64, 64], torch.nn.Tanh(), env, 5)
    h = net.head()
    assert isinstance(h, BinnedHead) and h.bins == 5 and h.adim == 3 and not net.is_tanh_mlp()
    assert h.low.dtype == np.float32 and np.array_equal(h.low, env.action_space.low) and np.array_equal(h.high, env.action_space.high)
    assert net.layer_sizes() == [15, 64, 64, 15]
    assert h.key() == _binned_net(5, [-1.0] * 3, [1.0] * 3).head().key()
    assert h.key() != _binned_net(11, [-1.0] * 3, [1.0] * 3).head().key()
    assert FeedForward([64, 64], torch.nn.Tanh(), env, 0.0).head() == 'tanh'
    assert FeedForward([64, 64], torch.nn.ReLU(), env, 0.0).head() is None
    assert FFBinned([64, 64], torch.nn.ReLU(), env, 5).head() is None
    assert FFIntegGausAction([8], torch.nn.Tanh(), SyntheticEnv(5, 4, 10), 0.0).head() is None
    comm, ranker = dist.world(), CenteredRanker()
    for e in (env, ClosedLoopEnv(15, 3, 20)):
        policy = Policy(FFBinned([64, 64], torch.nn.Tanh(), e, 5), 0.02, Adam(len(Policy.get_flat(net)), 0.01))
        assert es._can_fuse_step(comm, policy, BatchedRollout(e, 20), ranker)
        assert es._can_fuse_step(comm, policy, BatchedRollout(e, 20, archive=np.zeros((4, 2))), ranker) is False  # one objective
        assert not es._can_fuse_step(comm, policy, BatchedRollout(e, 20), EliteRanker(CenteredRanker(), 0.1))
        assert not es._can_fuse_step(comm, policy, lambda model: None, ranker)
    relu = FFBinned([64, 64], torch.nn.ReLU(), env, 5)
    assert not es._can_fuse_step(comm, Policy(relu, 0.02, Adam(len(Policy.get_flat(relu)), 0.01)), BatchedRollout(env, 20), ranker)
    # heads the kernels do not take exactly as FFBinned.forward computes them stay on the module's forward
    wide = FFBinned([64, 64], torch.nn.Tanh(), SyntheticEnv(376, 17, 20), 16)          # 272 outputs > 256
    assert wide.head() is None
    assert not es._can_fuse_step(comm, Policy(wide, 0.02, Adam(len(Policy.get_flat(wide)), 0.01)),
                                 BatchedRollout(SyntheticEnv(376, 17, 20), 20), ranker)
    assert FFBinned([64, 64], torch.nn.Tanh(), env, 1).head() is None                  # the reference divides by bins - 1
    f64 = SyntheticEnv(15, 3, 20)
    f64.action_space.low = f64.action_space.low.astype(np.float64)                      # the forward then rounds once, in float64
    assert FFBinned([64, 64], torch.nn.Tanh(), f64, 5).head() is None
    assert FFBinned([64, 64], torch.nn.Tanh(), SyntheticEnv(15, 16, 20), 16).head() is not None    # 256 outputs
    assert FFBinned([1000], torch.nn.Tanh(), env, 5).head() is None                     # beyond the float32 kernel's tiles


def _python_loop(net, env, T):
    """What run_model does for a policy it does not fuse: FFBinned.forward and env.step at every step."""
    rews = []
    with torch.no_grad():
        ob = env.reset()
        for _ in range(T):
            a = net(torch.from_numpy(np.asarray(ob)).float(), rs=None)
            ob, r, _, _ = env.step(a.numpy())
            rews.append(r)
    return rews


def test_run_model_keeps_uncovered_binned_policies_in_the_python_loop():
    """A binned policy the kernels do not cover (17 x 16 = 272 outputs) runs through run_model and BatchedRollout's per-call
    fit_fn in the python loop, as before binned policies were fused (no device is touched), and the oracle's binned loop gives
    the same rewards on both envs."""
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    from es_pytorch_b200.nn.nn import FFBinned
    T = 12
    for closed in (False, True):
        env = (ClosedLoopEnv if closed else SyntheticEnv)(376, 17, T)
        torch.manual_seed(2)
        net = FFBinned([64, 64], torch.nn.Tanh(), env, 16)
        assert net.head() is None
        rews, behv, obs, step = run_model(net, env, T)
        assert len(rews) == T and step == T - 1 and len(behv) == 3 * T
        assert rews == _python_loop(net, env, T)
        res = BatchedRollout(env, T, coins_per_eval=0)(net, False)
        assert res.result[0] == sum(rews)
        sizes = net.layer_sizes()
        layers = orc.unflatten(Policy.get_flat(net).astype(np.float32), orc.layer_dims(sizes[0], sizes[1:-1], sizes[-1]))
        spec = (orc.ClosedLoopEnvSpec if closed else orc.SyntheticEnvSpec)(376, 17, T)
        want, _, _, _ = orc.run_model(spec, layers, np.zeros(376), np.ones(376), 5.0, T,
                                      binned=(16, env.action_space.low, env.action_space.high))
        assert np.array_equal(np.array(rews), np.array(want))


def test_binned_entry_points_are_declared_bound_and_exported():
    from es_pytorch_b200 import _lib, build
    build.build()
    hdr = open(os.path.join(ROOT, 'include', 'es_b200.h')).read()
    lib = _lib.load()
    for name in ('es_rollout_openloop_binned', 'es_rollout_closedloop_mlp_binned', 'es_rollout_closedloop_mlp_binned_plan'):
        assert re.search(r'\b%s\s*\(' % name, hdr) and name in _lib.SIGNATURES and hasattr(lib, name), name
    # the head arguments follow the existing ones
    assert _lib.SIGNATURES['es_rollout_openloop_binned'][1][:19] == _lib.SIGNATURES['es_rollout_openloop'][1][:19]
    assert _lib.SIGNATURES['es_rollout_closedloop_mlp_binned'][1][:30] == _lib.SIGNATURES['es_rollout_closedloop_mlp'][1][:30]
    assert lib.es_abi_version() == 1


def _nvcc():
    import shutil
    from es_pytorch_b200 import build
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


def _ptxas_log(src, tmp):
    from es_pytorch_b200 import build
    cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
           '-o', os.path.join(tmp, os.path.basename(src) + '.o'), os.path.join(build.CSRC, src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    return log


def _props(log, kernel):
    return re.findall(r'Function properties for (\S*%s\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads' % kernel, log)


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_binned_open_loop_kernels_compile_for_sm90a_without_spills():
    """The binned instantiations (F32: weights in shared memory and in the global scratch; the TC3 tensor-core kernel) have
    their own names, spill nothing, and leave the tanh instantiations' counts as they were.  The closed-loop cluster kernel's
    binned instantiations are checked with its other variants in test_host_ptxas_closed_wide.py."""
    with tempfile.TemporaryDirectory() as tmp:
        f32 = _ptxas_log('rollout_f32.cu', tmp)
        tcw = _ptxas_log('rollout_tcw.cu', tmp)
    for log in (f32, tcw):
        for code in ('C7520', 'C7511', 'C7512', 'C7507'):
            assert code not in log, log
    for log, kernel, n in ((f32, 'rollout_f32_binned_kernel', 2), (f32, 'rollout_f32_kernel', 2),
                           (tcw, 'rollout_tcw_binned_kernel', 1), (tcw, 'rollout_tcw_kernel', 4)):
        props = _props(log, kernel)
        assert len(props) == n, (kernel, log)
        for name, _, st, ld in props:
            assert st == '0' and ld == '0', f'{name}: {st} bytes spill stores, {ld} bytes spill loads'


HARNESS = r'''
#include <stdarg.h>
#include <stdio.h>
#include "%s"
static char g_msg[512];
void es_set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_msg, sizeof g_msg, fmt, ap); va_end(ap); }
static void one(const char* name, const int* d, int nl, int band, int bins) {
    int C = 0, Ct = 0; size_t smem = 0, smem_t = 0;
    const int rc = es_closedw_binned_plan(d, nl, band, bins, &C, &smem);
    char msg[512];
    snprintf(msg, sizeof msg, "%%s", rc ? g_msg : "-");
    int dt[8];
    for (int i = 0; i <= nl; ++i) dt[i] = d[i];
    dt[nl] = d[nl] / (bins > 0 ? bins : 1);
    es_closedw_plan(dt, nl, band, &Ct, &smem_t);
    printf("%%s rc %%d C %%d smem %%zu tanh_smem %%zu msg %%s\n", name, rc, C, smem, smem_t, msg);
}
int main() {
    const int a[] = {15, 256, 256, 15}, b[] = {15, 256, 256, 33}, c[] = {17, 256, 256, 256, 30}, e[] = {28, 128, 256, 256, 128, 88},
              f[] = {8, 16, 16, 10}, g[] = {8, 16, 16, 258}, h[] = {8, 16, 16, 129};
    one("simple5", a, 3, 8, 5); one("simple11", b, 3, 8, 11); one("obj5", c, 4, 8, 5); one("flagrun11", e, 5, 8, 11);
    one("small", f, 3, 8, 5); one("wide", g, 3, 8, 2); one("bins1", h, 3, 8, 1);
    return 0;
}
'''


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_binned_closed_plan_on_the_host():
    """es_closedw_binned_plan: the shipped configs' trunks with bins 5 and 11 fit; a small shape takes a cluster of one CTA;
    adim * bins > 256 and bins < 2 are refused."""
    from es_pytorch_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, 'plan.cu')
        with open(src, 'w') as fh:
            fh.write(HARNESS % os.path.join(build.CSRC, 'rollout_closedw.cu').replace('\\', '/'))
        exe = os.path.join(tmp, 'plan')
        res = subprocess.run([_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-std=c++17', '-o', exe, src],
                             capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120).stdout
    plans = {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4)), int(m.group(5)), m.group(6))
             for m in re.finditer(r'^(\w+) rc (-?\d+) C (\d+) smem (\d+) tanh_smem (\d+) msg (.*)$', out, re.M)}
    for name in ('simple5', 'simple11', 'obj5', 'flagrun11', 'small'):
        rc, C, smem, _, _ = plans[name]
        assert rc == 0 and C >= 1 and smem <= 227 * 1024 - 1024, (name, plans[name])
    assert plans['small'][1] == 1
    assert plans['wide'][0] != 0 and '256' in plans['wide'][4]
    assert plans['bins1'][0] != 0 and 'bins' in plans['bins1'][4]
