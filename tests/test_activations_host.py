"""CPU (no GPU): policies with ReLU, leaky-ReLU, ELU and sigmoid activations.

* ``BaseNet.activation`` finds the one activation a plain-forward FeedForward applies after every layer, with LeakyReLU's slope
  and ELU's alpha rounded to float32, and None for everything the kernels do not evaluate; ``head`` / ``is_tanh_mlp`` do not
  move;
* the fused route is opt-in: a default BatchedRollout keeps today's decisions, ``fuse_activations=True`` fuses exactly the
  networks ``activation`` describes;
* the Activation alone rebuilds the network's arithmetic: a forward through the torch module it names equals the module's own
  forward bit for bit (what the GPU tests take as the float32 truth);
* the float64 truths of the GPU tests (tests/f64_rollout.py, tests/closed_f64.py) with each activation's form are the
  float32 forward through torch's modules to float32 rounding, and the forms are torch's in float64;
* the new sources compile for sm_90a without spills or serialised wgmma, within the closed-loop plan's static shared memory;
* the entry points are declared, bound and exported, and the kinds match the header.
"""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _env(obs=17, act=6, T=20, closed=False):
    from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
    return (ClosedLoopEnv if closed else SyntheticEnv)(obs, act, T)


def torch_module(act):
    """The torch module an ``nn.Activation`` stands for."""
    return {_lib.ES_ACT_TANH: lambda p: torch.nn.Tanh(), _lib.ES_ACT_RELU: lambda p: torch.nn.ReLU(),
            _lib.ES_ACT_LEAKY_RELU: lambda p: torch.nn.LeakyReLU(p), _lib.ES_ACT_ELU: lambda p: torch.nn.ELU(p),
            _lib.ES_ACT_SIGMOID: lambda p: torch.nn.Sigmoid()}[act.kind](act.param)


def mlp_forward(theta, layer_sizes, x, act):
    """Linear + activation after every layer from the flat state-dict parameters, in float32 through torch's own modules."""
    m = torch_module(act)
    a, off = torch.as_tensor(x, dtype=torch.float32), 0
    for fi, fo in zip(layer_sizes[:-1], layer_sizes[1:]):
        w = torch.as_tensor(theta[off:off + fi * fo], dtype=torch.float32).reshape(fo, fi)
        b = torch.as_tensor(theta[off + fi * fo:off + fi * fo + fo], dtype=torch.float32)
        a = m(torch.nn.functional.linear(a, w, b))
        off += fi * fo + fo
    return a


KINDS = [(torch.nn.Tanh(), _lib.ES_ACT_TANH, 0.0), (torch.nn.ReLU(), _lib.ES_ACT_RELU, 0.0),
         (torch.nn.LeakyReLU(0.1), _lib.ES_ACT_LEAKY_RELU, float(np.float32(0.1))),
         (torch.nn.ELU(0.7), _lib.ES_ACT_ELU, float(np.float32(0.7))), (torch.nn.ELU(), _lib.ES_ACT_ELU, 1.0),
         (torch.nn.Sigmoid(), _lib.ES_ACT_SIGMOID, 0.0)]


@pytest.mark.parametrize('module,kind,param', KINDS, ids=lambda v: type(v).__name__ if isinstance(v, torch.nn.Module) else None)
def test_activation_of_each_kind(module, kind, param):
    from es_pytorch_b200.nn.nn import Activation, FeedForward
    env = _env()
    net = FeedForward([64, 64], module, env, 0.0)
    act = net.activation()
    assert act == Activation(kind, param) and type(act.param) is float
    assert act.param == float(np.float32(act.param))                        # carried as the float32 value
    assert act.key() == ('activation', kind, param)
    # head / is_tanh_mlp are what they were: only tanh stacks are fused by default
    assert net.head() == ('tanh' if kind == _lib.ES_ACT_TANH else None)
    assert net.is_tanh_mlp() == (kind == _lib.ES_ACT_TANH)


def test_slope_and_alpha_are_rounded_to_float32():
    from es_pytorch_b200.nn.nn import FeedForward
    env = _env()
    for m, p in ((torch.nn.LeakyReLU(0.3), 0.3), (torch.nn.ELU(1.1), 1.1)):
        a = FeedForward([64], m, env, 0.0).activation()
        assert a.param == float(np.float32(p)) and a.param != p
    assert FeedForward([64], torch.nn.LeakyReLU(float('inf')), env, 0.0).activation() is None
    assert FeedForward([64], torch.nn.ELU(float('nan')), env, 0.0).activation() is None
    # keys tell parameters apart that differ in float32, and only those
    k = lambda s: FeedForward([64], torch.nn.LeakyReLU(s), env, 0.0).activation().key()
    assert k(0.1) != k(0.2) and k(0.1) == k(float(np.float32(0.1)))


def test_other_networks_have_no_activation():
    from es_pytorch_b200.nn.nn import FeedForward, FFBinned, FFIntegGausAction, FFIntegGausActionMulti
    env = _env()
    mixed = FeedForward([64, 64], torch.nn.ReLU(), env, 0.0)
    mixed.model[3] = torch.nn.Tanh()
    assert mixed.activation() is None
    slopes = FeedForward([64, 64], torch.nn.LeakyReLU(0.1), env, 0.0)
    slopes.model[3] = torch.nn.LeakyReLU(0.2)
    assert slopes.activation() is None

    class MyReLU(torch.nn.ReLU):
        pass

    class MyNet(FeedForward):
        def forward(self, inp, **kwargs):
            return super().forward(inp, **kwargs) * 2

    assert FeedForward([64], MyReLU(), env, 0.0).activation() is None
    assert FeedForward([64], torch.nn.GELU(), env, 0.0).activation() is None
    assert MyNet([64], torch.nn.ReLU(), env, 0.0).activation() is None
    assert FFBinned([64, 64], torch.nn.ReLU(), env, 5).activation() is None
    assert FFBinned([64, 64], torch.nn.Tanh(), env, 5).activation() is None
    assert FFIntegGausAction([8], torch.nn.ReLU(), _env(5, 4), 0.0).activation() is None
    assert FFIntegGausActionMulti([8], torch.nn.ELU(), _env(5, 4), 0.0).activation() is None


@pytest.mark.parametrize('closed', [False, True])
def test_the_device_route_is_opt_in(closed):
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.nn import Activation, FeedForward, FFBinned
    from es_pytorch_b200.nn.optimizers import Adam
    from es_pytorch_b200.utils.rankers import CenteredRanker, EliteRanker
    env = _env(closed=closed)
    comm, ranker = dist.world(), CenteredRanker()
    pol = lambda net: Policy(net, 0.02, Adam(len(Policy.get_flat(net)), 0.01))
    off, on = BatchedRollout(env, 20), BatchedRollout(env, 20, fuse_activations=True)
    assert off.fuse_activations is False and on.fuse_activations is True
    for m, _, _ in KINDS[1:]:
        net = FeedForward([64, 64], m, env, 0.0)
        assert not es._can_fuse_step(comm, pol(net), off, ranker)            # today's route: the python loop
        assert es._fused_policy(net, off) is None and off.fused_activation(net) is None
        assert es._can_fuse_step(comm, pol(net), on, ranker)
        assert es._fused_policy(net, on) == ('tanh', net.activation()) and on.fused_activation(net) == net.activation()
        assert not es._can_fuse_step(comm, pol(net), on, EliteRanker(CenteredRanker(), 0.1))     # the ranker still decides
    tanh = FeedForward([64, 64], torch.nn.Tanh(), env, 0.0)
    for b in (off, on):                                                       # tanh keeps its route either way
        assert es._can_fuse_step(comm, pol(tanh), b, ranker) and es._fused_policy(tanh, b) == ('tanh', None)
    relu_binned = FFBinned([64, 64], torch.nn.ReLU(), env, 5)
    assert not es._can_fuse_step(comm, pol(relu_binned), on, ranker)          # binned heads stay tanh-only
    assert on.fused_activation(relu_binned) is None
    assert Activation(_lib.ES_ACT_TANH, 0.0) == tanh.activation() and on.fused_activation(tanh) is None


def test_python_loop_stays_the_default_route():
    """Without the flag a ReLU policy's BatchedRollout call and run_model run the python loop (no device here), with the flag
    the call goes to the device."""
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    from es_pytorch_b200.nn.nn import FeedForward
    env = _env(T=8)
    torch.manual_seed(0)
    net = FeedForward([16, 16], torch.nn.ReLU(), env, 0.0)
    rews, _, _, _ = run_model(net, env, 8, None)
    assert len(rews) == 8                                                     # one reward per step: the python loop
    got = BatchedRollout(env, 8, coins_per_eval=0)(net, False)
    assert got.result == np.sum(rews)
    if not torch.cuda.is_available():
        with pytest.raises(Exception):
            BatchedRollout(env, 8, coins_per_eval=0, fuse_activations=True)(net, False)


@pytest.mark.parametrize('module,kind,param', KINDS, ids=lambda v: type(v).__name__ if isinstance(v, torch.nn.Module) else None)
def test_activation_rebuilds_the_network_forward(module, kind, param):
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.nn.nn import FeedForward
    env = _env()
    torch.manual_seed(1)
    net = FeedForward([64, 32], module, env, 0.0)
    x = torch.randn(50, env.observation_space.shape[0]) * 3
    with torch.no_grad():
        want = net.model(x).numpy()
    got = mlp_forward(Policy.get_flat(net), net.layer_sizes(), x, net.activation()).numpy()
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def _nvcc():
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


def _ptxas_log(name, tmp):
    cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
           '-o', os.path.join(tmp, name + '.o'), os.path.join(build.CSRC, name + '.cu')]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    return log


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_tcw_activation_kernels_compile_without_spills():
    # (the closed-loop cluster kernel's activation instantiations are checked in test_host_ptxas_closed_wide.py)
    with tempfile.TemporaryDirectory() as tmp:
        tcw = _ptxas_log('rollout_tcw_act', tmp)
    spill = r'Function properties for (\S*%s\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads'
    props = re.findall(spill % 'rollout_tcwa_kernel', tcw)
    assert len(props) == 8, tcw                                 # 4 kinds x with / without action noise
    for name, stack, st, ld in props:
        assert stack == '0' and st == '0' and ld == '0', (name, stack, st, ld)
    for code in ('C7520', 'C7512', 'C7511', 'C7507'):           # wgmma serialised by ptxas
        assert code not in tcw, code


def test_activation_entry_points_are_declared_bound_and_built():
    build.build()
    hdr = open(os.path.join(ROOT, 'include', 'es_b200.h')).read()
    lib = _lib.load()
    for name in ('es_rollout_openloop_activation', 'es_rollout_closedloop_mlp_activation',
                 'es_rollout_closedloop_mlp_activation_plan'):
        assert re.search(r'\b%s\s*\(' % name, hdr) and name in _lib.SIGNATURES and hasattr(lib, name)
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    kinds = {k: int(v) for k, v in re.findall(r'#define\s+(ES_ACT_\w+)\s+(\d+)', hdr)}
    assert kinds == {k: getattr(_lib, k) for k in ('ES_ACT_TANH', 'ES_ACT_RELU', 'ES_ACT_LEAKY_RELU', 'ES_ACT_ELU',
                                                    'ES_ACT_SIGMOID')}
    assert kinds['ES_ACT_TANH'] == 0                             # a zero-initialised call is a tanh call
    for src in ('rollout_tcw_act.cu', 'rollout_closedw.cu'):
        assert src in build.SOURCES
    for h in ('rollout_tcw.cuh', 'rollout_closedw.cuh'):
        assert h in build.HEADERS


def _f64_helpers():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import closed_f64
    import f64_rollout
    return closed_f64, f64_rollout


@pytest.mark.parametrize('E,noisy', [(1, False), (3, True)])
def test_float64_truth_with_tanh_is_the_tanh_truth(E, noisy):
    """Open loop: the float64 truth with every kind's form is the float32 forward through torch's own modules to float32
    rounding (fitness and behaviour, per evaluation).  Closed loop: tanh given per layer is the default bit for bit, and
    another activation changes the policy, not the env: a ReLU truth differs."""
    from es_pytorch_b200.nn.nn import Activation
    closed_f64, f64_rollout = _f64_helpers()
    rs = np.random.RandomState(4)
    sizes, T, n = [9, 16, 12, 4], 7, 3
    P = f64_rollout.n_params(sizes)
    table = rs.randn(P + 100).astype(np.float32)
    theta = (rs.randn(P) * 0.3).astype(np.float32)
    idx = rs.randint(0, 100, size=n)
    obsn = rs.randn(T, sizes[0]).astype(np.float32)
    rew = rs.randn(T, sizes[-1]).astype(np.float32)
    noise = (rs.randn(n, 2, E, T, sizes[-1]) * 0.1).astype(np.float32) if noisy else None
    c, cols = rew.astype(np.float64), [j % sizes[-1] for j in range(3)]
    for _, kind, param in KINDS:
        act = Activation(kind, param)
        fit, behv, mass, mag = f64_rollout.rollout_f64(table, idx, theta, 0.02, sizes, obsn, rew, 0.05, noise, E,
                                                       activation=f64_rollout.form(act))
        for k in range(n):
            for s, sign in enumerate((1.0, -1.0)):
                w = f64_rollout.perturbed(table, idx[k], theta, 0.02, sign).astype(np.float32)
                a = mlp_forward(w, sizes, obsn, act).numpy().astype(np.float64)
                nz = np.zeros((1, T, sizes[-1])) if noise is None else noise[k, s].astype(np.float64)
                f32_fit = np.mean([((a + z) * c).sum() for z in nz])
                f32_behv = 0.05 * (a + nz[-1])[:, cols].sum(axis=0)
                assert abs(f32_fit - fit[s, k]) <= 1e-6 * mass[s, k], (kind, k, s)
                assert np.all(np.abs(f32_behv - behv[s, k]) <= 1e-6 * mag[s, k]), (kind, k, s)
    band = 4
    args = (table, idx, theta, 0.02, sizes, rs.randn(sizes[0]) * 0.1, 0.5 + rs.rand(sizes[0]), 1.0,
            rs.randn(sizes[0]).astype(np.float32), (rs.randn(band, sizes[0]) * 0.4).astype(np.float32),
            (rs.randn(sizes[-1], sizes[0]) * 0.4).astype(np.float32), rew, 0.05)
    want = closed_f64.truth(*args, act_noise=noise, episodes=E)
    got = closed_f64.truth(*args, act_noise=noise, episodes=E, activation=[np.tanh] * (len(sizes) - 1))
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    relu = closed_f64.truth(*args, act_noise=noise, episodes=E, activation=f64_rollout.relu)
    assert not np.allclose(relu['fit'], want['fit'])


def test_float64_activation_forms_match_torch_in_float64():
    _, f64_rollout = _f64_helpers()
    z = np.linspace(-30, 30, 2001)
    t = torch.from_numpy(z)
    for f, m in ((f64_rollout.relu, torch.nn.ReLU()), (f64_rollout.leaky_relu(0.1), torch.nn.LeakyReLU(float(np.float32(0.1)))),
                 (f64_rollout.elu(0.7), torch.nn.ELU(float(np.float32(0.7)))), (f64_rollout.sigmoid, torch.nn.Sigmoid())):
        np.testing.assert_allclose(f(z), m(t).numpy(), rtol=1e-14, atol=1e-300)
