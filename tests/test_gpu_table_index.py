"""Every kernel that reads a noise slice reports an index outside the table.

NoiseTable.get asserts ``len(self) > i + size`` (src/core/noisetable.py:34).  On the device every reader takes its slice
through es_checked_slice (common.cuh), which replaces a bad index by slice 0, so no load leaves the table, and sets the ctx's
error word; the next entry point, or ``Engine.sync``, raises "noise index outside the table" and clears the word.  Each case
below is a valid call of one reader with one index set to ``L - P`` (the first inadmissible slice) and then to -1: the call or
the sync after it must raise, and the next valid call on the same engine must succeed.  If a reader lost its reporting
site, a bad index would silently read slice 0 and the results would look like any others."""
import numpy as np
import pytest
import torch

from es_pytorch_b200 import _lib
from es_pytorch_b200._lib import EsLibraryError
from es_pytorch_b200.nn.nn import Activation, BinnedHead
from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu

F32, TC, TC3 = _lib.ES_ROLLOUT_F32, _lib.ES_ROLLOUT_TC, _lib.ES_ROLLOUT_TC3
RELU = Activation(_lib.ES_ACT_RELU, 0.0)


def _n_params(sizes):
    return orc.n_params(orc.layer_dims(sizes[0], sizes[1:-1], sizes[-1]))


def _inputs(eng, sizes, n, seed=0):
    rs = np.random.RandomState(seed)
    P = _n_params(sizes)
    L = P + 20_000
    d = eng.to_device
    return P, L, d(rs.randn(L).astype(np.float32)), d((rs.randn(P) * 0.1).astype(np.float32)), \
        rs.randint(0, L - P, size=n).astype(np.int64)


def _open(sizes, n, mode=F32, head=None, activation=None, env=None):
    """A call of the open-loop rollout: (P, L, good indices, run(idx))."""
    def make(eng):
        P, L, table, theta, idx = _inputs(eng, sizes, n)
        T = 40
        act = head.adim if head is not None else sizes[-1]
        rs = np.random.RandomState(1)
        obsn = eng.to_device(np.clip(rs.randn(T, sizes[0]), -5, 5).astype(np.float32))
        rew = eng.to_device(rs.randn(T, act).astype(np.float32))

        def run(ix):
            fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
            behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
            eng.rollout(table, eng.to_device(ix), theta, 0.02, sizes, obsn, rew, 0.05, fit[0], fit[1], 1, behv[0], behv[1],
                        mode, head=head, activation=activation)
        return P, L, idx, run
    return make


def _closed(sizes, n, head=None, activation=None, one_cta=False):
    """A call of the closed-loop rollout (rollout_closed_mlp); ``one_cta``: the plan must be rollout_closed.cu's kernel."""
    def make(eng):
        P, L, table, theta, idx = _inputs(eng, sizes, n)
        act = head.adim if head is not None else sizes[-1]
        spec = orc.ClosedLoopEnvSpec(sizes[0], act, 30, band=8)
        C = eng.closed_mlp_plan(sizes, spec.band, head, activation)[0]
        assert (C == 0) == one_cta, C
        d = eng.to_device
        mean, std = d(np.zeros(sizes[0])), d(np.ones(sizes[0]))
        obs0, env_a, env_b = d(spec.obs_stream[0].copy()), d(np.ascontiguousarray(spec.env_a.T)), d(np.ascontiguousarray(spec.env_b.T))
        rew = d(spec.rew_vec)

        def run(ix):
            fit = torch.zeros(2, n, dtype=torch.float64, device=eng.device)
            behv = torch.zeros(2, n, 3, dtype=torch.float32, device=eng.device)
            eng.rollout_closed_mlp(table, eng.to_device(ix), theta, 0.02, sizes, mean, std, 5.0, obs0, env_a, env_b, rew,
                                   spec.pos_scale, fit[0], fit[1], 1, behv[0].view(-1), behv[1].view(-1), head=head,
                                   activation=activation)
        return P, L, idx, run
    return make


def _perturb(eng):
    P, L, table, theta, idx = _inputs(eng, [17, 64, 64, 6], 5)
    return P, L, idx, lambda ix: eng.perturb(theta, table, eng.to_device(ix), 0.02)


def _reconstruct(eng):
    P, L, table, _, idx = _inputs(eng, [17, 64, 64, 6], 300)
    w = eng.to_device(np.random.RandomState(2).rand(300).astype(np.float32))
    return P, L, idx, lambda ix: eng.grad_reconstruct(table, eng.to_device(ix), w, P)


def _f32x(eng):
    """The packed-FMA kernel (rollout_f32x.cu) at more pairs than CTAs: CTA 0 runs pairs 0 and sm_count."""
    return _open([17, 64, 64, 6], eng.sm_count + 3)(eng)


BINNED = BinnedHead(5, np.float32([-1.0, 0.0, 0.5]), np.float32([1.0, 2.0, 0.75]))

# (id, builder, which pair gets the bad index (None: pair 1), environment)
CASES = [
    ('perturb', _perturb, None, {}),
    ('grad_reconstruct', _reconstruct, None, {}),
    ('f32_general_shared_weights', _open([17, 64, 64, 6], 4), None, {'ES_F32_GENERAL': '1'}),
    ('f32_general_staged_weights', _open([15, 256, 256, 3], 4), None, {}),
    ('f32x_first_pair', _f32x, 0, {}),
    ('f32x_later_pair', _f32x, 'sm', {}),
    ('tc2_tc', _open([17, 64, 64, 6], 6, TC), None, {}),
    ('tc2_tc3', _open([17, 64, 64, 6], 6, TC3), None, {}),
    ('tc2_tc_shadows', _open([24, 64, 64, 6], 6, TC), None, {}),
    ('tc2_tc3_shadows', _open([24, 64, 64, 6], 6, TC3), None, {}),
    ('tcw_act_relu_tc3', _open([15, 256, 256, 3], 4, TC3, activation=RELU), None, {}),
    ('binned_open_f32', _open([15, 64, 64, 15], 4, F32, head=BINNED), None, {}),
    ('binned_open_tc3', _open([15, 64, 64, 15], 4, TC3, head=BINNED), None, {}),
    ('closed_one_cta', _closed([17, 64, 64, 6], 3, one_cta=True), None, {}),
    ('closed_wide', _closed([15, 256, 256, 3], 3), None, {}),
    ('closed_activation', _closed([17, 64, 64, 6], 3, activation=RELU), None, {}),
    ('closed_binned', _closed([15, 64, 64, 15], 3, head=BINNED), None, {}),
]


@pytest.mark.parametrize('bad', ['L-P', '-1'])
@pytest.mark.parametrize('name,make,pair,env', CASES, ids=[c[0] for c in CASES])
def test_index_outside_the_table_is_reported(eng, monkeypatch, name, make, pair, env, bad):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    P, L, idx, run = make(eng)
    pair = {None: 1, 'sm': eng.sm_count}.get(pair, pair)
    eng.sync()
    wrong = idx.copy()
    wrong[pair] = L - P if bad == 'L-P' else -1
    with pytest.raises(EsLibraryError, match='outside the table'):
        run(wrong)
        eng.sync()
    run(idx)                                   # the word was cleared: a valid call goes through, and reports nothing
    eng.sync()
    idx[pair] = L - P - 1                      # the last admissible slice is not reported
    run(idx)
    eng.sync()
