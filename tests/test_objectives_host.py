"""CPU (no GPU): the single-objective adaptors through BatchedRollout -- which combinations it accepts, the objective columns it
announces, which of them es.step fuses, the one-step MeanRewardResult refusal, the python-loop route's results -- and the
objective kernel's entry point and compilation for sm_90a."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _classes():
    from es_pytorch_b200.gym import training_result as tr
    return tr.RewardResult, tr.MeanRewardResult, tr.DistResult, tr.XDistResult, tr.NSResult, tr.NSRResult


def _env(T=20):
    from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
    return SyntheticEnv(17, 6, T)


ARCHIVE = np.random.RandomState(3).randn(6, 2)


def test_batched_rollout_accepts_the_six_adaptors_and_refuses_the_rest():
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.training_result import MultiAgentTrainingResult, TrainingResult
    Reward, Mean, Dist, XDist, NS, NSR = _classes()
    env = _env()
    # the defaults keep the rule of the two adaptors the fused route had before
    assert BatchedRollout(env, 20).result is Reward
    assert BatchedRollout(env, 20, archive=ARCHIVE).result is NSR
    for cls in (Reward, Mean, Dist, XDist):
        b = BatchedRollout(env, 20, result=cls)
        assert b.result is cls and b.n_obj == 1
        with pytest.raises(ValueError, match='archive'):
            BatchedRollout(env, 20, archive=ARCHIVE, result=cls)          # an archive with a non-novelty adaptor
    for cls, n_obj in ((NS, 1), (NSR, 2)):
        assert BatchedRollout(env, 20, archive=ARCHIVE, result=cls).n_obj == n_obj
        with pytest.raises(ValueError, match='archive'):
            BatchedRollout(env, 20, result=cls)                           # novelty without an archive
        with pytest.raises(ValueError, match='episodes'):
            BatchedRollout(env, 20, archive=ARCHIVE, result=cls, episodes=2)

    class MyResult(Reward):
        pass
    an_instance = Reward([1.0], [0.0] * 3, np.zeros((1, 17)), 0)
    for bad in (MultiAgentTrainingResult, TrainingResult, MyResult, 'DistResult', an_instance, type(None)):
        with pytest.raises(ValueError, match='result must be one of'):
            BatchedRollout(env, 20, result=bad)


def _policy(env, act=torch.nn.Tanh()):
    from es_pytorch_b200.core.policy import Policy
    from es_pytorch_b200.nn.nn import FeedForward
    from es_pytorch_b200.nn.optimizers import Adam
    net = FeedForward([32, 32], act, env, 0.0)
    return Policy(net, 0.02, Adam(len(Policy.get_flat(net)), 0.01))


def test_single_objective_adaptors_fuse_with_the_plain_rankers():
    from es_pytorch_b200 import dist
    from es_pytorch_b200.core import es
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.utils import rankers as R
    Reward, Mean, Dist, XDist, NS, NSR = _classes()
    env = _env()
    policy, comm = _policy(env), dist.world()
    for cls in (Mean, Dist, XDist, NS):
        fit_fn = BatchedRollout(env, 20, archive=ARCHIVE if cls is NS else None, result=cls)
        assert es._can_fuse_step(comm, policy, fit_fn, R.CenteredRanker()), cls
        assert es._can_fuse_step(comm, policy, fit_fn, R.SemiCenteredRanker()), cls
        assert not es._can_fuse_step(comm, policy, fit_fn, R.EliteRanker(R.CenteredRanker(), 0.1)), cls
        assert not es._can_fuse_step(comm, policy, fit_fn, R.MaxNormalizedRanker()), cls
    # MultiObjectiveRanker asserts two columns (rankers.py:114): novelty alone is one
    ns = BatchedRollout(env, 20, archive=ARCHIVE, result=NS)
    assert not es._can_fuse_step(comm, policy, ns, R.MultiObjectiveRanker(R.CenteredRanker(), 0.5))
    assert es._can_fuse_step(comm, policy, BatchedRollout(env, 20, archive=ARCHIVE, result=NSR),
                             R.MultiObjectiveRanker(R.CenteredRanker(), 0.5))


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def test_one_step_mean_reward_raises_before_anything_runs(monkeypatch):
    """MeanRewardResult divides by steps, the last loop index: 0 for a one-step episode.  es.test_params and es.step raise the
    reference's ZeroDivisionError before a generation is built (no engine, so nothing is launched)."""
    from es_pytorch_b200 import dist, engine
    from es_pytorch_b200.core import es
    from es_pytorch_b200.core.noisetable import NoiseTable
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.nn.obstat import ObStat
    from es_pytorch_b200.utils.rankers import CenteredRanker
    from es_pytorch_b200.utils.reporters import Reporter
    Reward, Mean = _classes()[:2]

    def no_engine(*a, **k):
        raise AssertionError('the device was reached')
    monkeypatch.setattr(engine, 'get_engine', no_engine)
    monkeypatch.setattr(es, 'get_engine', no_engine)
    env = _env(1)
    policy = _policy(env)
    nt = NoiseTable(len(policy), np.zeros(len(policy) + 100, dtype=np.float32))
    fit_fn = BatchedRollout(env, 1, result=Mean)
    rs = np.random.RandomState(0)
    before = rs.get_state()
    with pytest.raises(ZeroDivisionError):
        es.test_params(dist.world(), 2, policy, nt, ObStat(env.observation_space.shape, 0), fit_fn, rs)
    cfg = _Cfg(general=_Cfg(policies_per_gen=4, batch_size=500), policy=_Cfg(l2coeff=0.005))
    assert es._can_fuse_step(dist.world(), policy, fit_fn, CenteredRanker())
    with pytest.raises(ZeroDivisionError):
        es.step(cfg, dist.world(), policy, nt, env, fit_fn, rs, CenteredRanker(), Reporter())
    assert fit_fn._gen is None and np.array_equal(rs.get_state()[1], before[1]) and rs.get_state()[2] == before[2]
    # two steps have steps == 1: no refusal there (the device is then reached)
    with pytest.raises(AssertionError, match='device was reached'):
        es.test_params(dist.world(), 2, policy, nt, ObStat(env.observation_space.shape, 0),
                       BatchedRollout(_env(2), 2, result=Mean), rs)


def test_python_loop_route_builds_the_requested_adaptor():
    """A policy the fused kernels do not evaluate (ReLU) runs run_model's python loop on the host: the BatchedRollout's call
    returns the requested class, with the result the class computes from run_model's record."""
    from es_pytorch_b200.gym.batched import BatchedRollout
    from es_pytorch_b200.gym.gym_runner import run_model
    T = 12
    env = _env(T)
    torch.manual_seed(0)
    net = _policy(env, torch.nn.ReLU())._module
    rews, behv, _, steps = run_model(net, env, T, None)
    no_obs = np.array([np.zeros(env.observation_space.shape)])
    for cls in _classes():
        archive = ARCHIVE if cls.__name__.startswith('NS') else None
        got = BatchedRollout(env, T, coins_per_eval=0, archive=archive, result=cls)(net, False)
        assert type(got) is cls
        want = cls(rews, behv[-3:], no_obs, steps, ARCHIVE, 10) if archive is not None else cls(rews, behv, no_obs, steps)
        if archive is None:                       # the novelty adaptors' novelty runs on the device (utils.novelty)
            assert got.result == want.result, cls
    # the reference's one-step MeanRewardResult: built, and raising on the first .result access
    env1 = _env(1)
    got = BatchedRollout(env1, 1, coins_per_eval=0, result=_classes()[1])(_policy(env1, torch.nn.ReLU())._module, False)
    assert got.steps == 0
    with pytest.raises(ZeroDivisionError):
        got.result


def test_objective_entry_point_is_declared_bound_and_exported():
    from es_pytorch_b200 import _lib, build
    build.build()
    hdr = open(os.path.join(ROOT, 'include', 'es_b200.h')).read()
    lib = _lib.load()
    name = 'es_fitness_objective'
    assert re.search(r'\b%s\s*\(' % name, hdr) and name in _lib.SIGNATURES and hasattr(lib, name)
    # (ctx, kind, fit, fit_stride, behv, n, steps, stream)
    assert _lib.SIGNATURES[name] == (_lib._i32, [_lib._vp, _lib._i32, _lib._vp, _lib._i32, _lib._vp, _lib._i32, _lib._i32,
                                                 _lib._vp])
    assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    kinds = dict(re.findall(r'\b(ES_OBJ_\w+)\s*=\s*(\d+)', hdr))
    assert {k: int(v) for k, v in kinds.items()} == {'ES_OBJ_MEAN_REWARD': _lib.ES_OBJ_MEAN_REWARD,
                                                      'ES_OBJ_DIST': _lib.ES_OBJ_DIST, 'ES_OBJ_XDIST': _lib.ES_OBJ_XDIST}
    assert lib.es_abi_version() == 1


def _nvcc():
    from es_pytorch_b200 import build
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_objective_kernel_compiles_for_sm90a_without_spills():
    from es_pytorch_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
               '-o', os.path.join(tmp, 'objective.o'), os.path.join(build.CSRC, 'objective.cu')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    assert 'objective.cu' in build.SOURCES
    props = re.findall(r'Function properties for (\S*fitness_objective_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes '
                       r'spill stores, (\d+) bytes spill loads', log)
    assert len(props) == 1, log
    for name, frame, st, ld in props:
        assert frame == '0' and st == '0' and ld == '0', (name, frame, st, ld)
