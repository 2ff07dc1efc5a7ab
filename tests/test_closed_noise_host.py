"""CPU (no GPU): the closed-loop action-noise oracle, the new entry point's declaration and binding, and the noisy / episodic
closed-loop kernels' compilation for sm_90a."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import es_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBS, ACT, HID, T = 9, 3, (8, 8), 13          # T * ACT odd: the gaussian cache crosses episodes


def _problem(seed=3):
    dims = orc.layer_dims(OBS, HID, ACT)
    rs = np.random.RandomState(seed)
    theta = (rs.randn(orc.n_params(dims)) * 0.3).astype(np.float32)
    return orc.unflatten(theta, dims), orc.ClosedLoopEnvSpec(OBS, ACT, T, band=4)


@pytest.mark.parametrize('E', [1, 2, 5])
def test_noise_free_closed_oracle_is_one_episode(E):
    """Without noise (ac_std = 0, or no stream) E episodes are the single noise-free episode, values and stream state
    identical."""
    layers, spec = _problem()
    mean, std = np.full(OBS, 0.1), np.full(OBS, 0.9)
    want = orc.run_model(spec, layers, mean, std, 5.0, T)
    rs = np.random.RandomState(1)
    before = rs.get_state()
    for ac_std, r in ((0.0, rs), (0.05, None)):
        got = orc.run_model(spec, layers, mean, std, 5.0, T, ac_std=ac_std, rs=r, episodes=E)
        assert got[0] == want[0] and got[1] == want[1] and np.array_equal(got[2], want[2]) and got[3] == want[3]
    after = rs.get_state()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))          # no noise, no draw


@pytest.mark.parametrize('E', [1, 2, 3])
def test_closed_oracle_consumes_one_randn_call_per_evaluation(E):
    layers, spec = _problem()
    rs, ref = np.random.RandomState(7), np.random.RandomState(7)
    rs.randn(1); ref.randn(1)                                               # start with a cached gaussian
    rews, behv, obs, step = orc.run_model(spec, layers, np.zeros(OBS), np.ones(OBS), 5.0, T, ac_std=0.05, rs=rs, episodes=E)
    ref.randn(E * T * ACT)
    a, b = rs.get_state(), ref.get_state()
    assert np.array_equal(a[1], b[1]) and a[2:] == b[2:]                    # key, position, has_gauss and the cached value
    # the noise moves the trajectory, and the last episode is the one reported
    clean = orc.run_model(spec, layers, np.zeros(OBS), np.ones(OBS), 5.0, T)
    assert rews != clean[0] and not np.array_equal(obs, clean[2])
    assert len(rews) == T and step == T - 1 and len(behv) == 3 * T


def test_closed_test_params_runs_the_noisy_episodes():
    """es_test_params on the closed loop with action noise and two episodes: pair 0's + evaluation by hand."""
    _, spec = _problem()
    dims = orc.layer_dims(OBS, HID, ACT)
    P = orc.n_params(dims)
    rs = np.random.RandomState(3)
    table = rs.randn(P + 500).astype(np.float32)
    theta = (rs.randn(P) * 0.3).astype(np.float32)
    pos, neg, inds, _, _ = orc.es_test_params(table, theta, 0.05, dims, spec, [5], 2, np.zeros(OBS), np.ones(OBS), 5.0, T,
                                              coins_per_eval=1, ac_std=0.05, episodes=2)
    assert pos.shape == (2, 1) and neg.shape == (2, 1)
    r = np.random.RandomState(5)
    idx = orc.sample_idx(len(table), r, P)
    r.random()
    lay = orc.unflatten(orc.pheno_params(theta, 0.05, orc.table_get(table, idx, P)), dims)
    rews, _, _, _ = orc.run_model(spec, lay, np.zeros(OBS), np.ones(OBS), 5.0, T, ac_std=0.05, rs=r, episodes=2)
    assert inds[0] == idx and pos[0, 0] == sum(rews)


def test_closed_episodes_entry_point_is_declared_bound_and_exported():
    from es_pytorch_b200 import _lib, build
    build.build()
    hdr = open(os.path.join(ROOT, 'include', 'es_b200.h')).read()
    lib = _lib.load()
    name = 'es_rollout_closedloop_mlp_episodes'
    assert re.search(r'\b%s\s*\(' % name, hdr) and name in _lib.SIGNATURES and hasattr(lib, name)
    # es_rollout_closedloop_mlp's arguments, then act_noise and n_episodes before the stream
    args, base = _lib.SIGNATURES[name][1], _lib.SIGNATURES['es_rollout_closedloop_mlp'][1]
    assert args[:30] == base[:30] and args[30:] == [_lib._vp, _lib._i32, _lib._vp]
    assert lib.es_abi_version() == 1


def _nvcc():
    import shutil
    from es_pytorch_b200 import build
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


def _props(src, kernel, tmp):
    from es_pytorch_b200 import build
    cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
           '-o', os.path.join(tmp, src + '.o'), os.path.join(build.CSRC, src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    return {n: (int(st), int(ld)) for n, _, st, ld in re.findall(
        r'Function properties for (\S*%s\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads'
        % kernel, log)}


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_noisy_one_cta_kernels_compile_for_sm90a():
    """The noisy / episodic instantiations of the one-CTA kernel have their own names, and those for obs <= 32 and <= 128
    spill nothing.  The one-CTA kernel for obs > 128 holds 96 registers of layer-1 weights per thread; its noise-free
    instantiation already spills, and the noisy one may spill at most 64 bytes more.  The cluster kernel's noisy
    instantiations are checked with its other variants in test_host_ptxas_closed_wide.py."""
    with tempfile.TemporaryDirectory() as tmp:
        cl = _props('rollout_closed.cu', 'rollout_closed_noisy_kernel', tmp)
        cl0 = _props('rollout_closed.cu', 'rollout_closed_kernel', tmp)
    assert len(cl) == 3 and len(cl0) == 3, (cl, cl0)
    for name, (st, ld) in cl.items():
        if 'ILi12E' in name:
            base = next(v for n, v in cl0.items() if 'ILi12E' in n)
            assert st <= base[0] + 64 and ld <= base[1] + 64, (name, st, ld, base)
        else:
            assert st == 0 and ld == 0, (name, st, ld)
