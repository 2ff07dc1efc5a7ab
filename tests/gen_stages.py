"""Stage-by-stage judge of one captured ES generation (DeviceGeneration.run, or es.step on its fused route).

TEST INFRASTRUCTURE ONLY.  Nothing here launches a kernel: a ``Capture`` holds what the generation started from and what it
produced, and ``judge`` checks every stage against a reference computed from the DEVICE'S OWN INPUTS TO THAT STAGE, so that a
near-tie that flips one rank cannot cascade into the checks of later stages:

  1 draws       numpy's streams replayed in the reference's order (es_oracle.es_test_params): per pair ``sample_idx``, per
                evaluation its ``rs.random()`` coin (two raw words), then with action noise ``rs.randn(T act) ac_std``.  Indices,
                coin words and the end states (key, position, has_gauss) exact, the cached gaussian to 2 ulp, the action noise
                by test_gpu_noise_table._mismatches (equal, or one float32 ulp away next to a rounding midpoint);
  2 obstat      sum, sumsq, count and n_saved exactly against ObStatOracle fed, in evaluation order, with the replayed coins and
                ob_sum_sq_cnt(obs_stream[1:T+1]);
  3 normalise   the normalised observations bit for bit against orc.normalise_obs with the generation's mean / std;
  4 fitness     every evaluation against float64 (``fitness_truth``: torch.float64 on the tensors' device, from the device's
                indices, theta, normalised observations and action noise, with the policy's activation
                ``Capture.activation`` in tests/f64_rollout.py's forms), judged by test_gpu_rollout_f64._check (EVAL_REL of
                the reward mass per evaluation, RMS_BOUND of the spread -- test_gpu_activations.RMS with an activation --,
                behaviours within float32 rounding); the float64 truth tied to the plain CPU reference
                tests/f64_rollout.rollout_f64 (with the activation) on sampled pairs to TIE_REL of the mass;
  5 novelty     (archive) bit for bit against orc.novelty of the device's behaviours, in column 1 of the [pos|neg][k][2] rows;
  6 weights     bit for bit against orc.centered_ranker / orc.moo_ranker on the device's fitness, n_ranked equal; and against
                the ranks of the float64 truth: how many ranks differ, the largest shift and the largest |dw| (bounded by
                the caller: they depend on the rollout arithmetic and the population);
  7 gradient    gsum against the float64 sum_k w_k eps_k of the device's weights and indices: rc_f64.truth_device / judge with
                rc_layout(P, K, sm), unchanged;
  8 optimizer   theta', m', v' bit for bit against orc.AdamOracle applied in float32 to the device's gsum and theta.

Episodes (``Capture.episodes`` = E): every evaluation draws E T act gaussians after its coin, the E episodes back to back;
its fitness is sum_t (r_1t + ... + r_Et) / E and its behaviour the last episode's.  Objectives (``Capture.objective``):
'reward' (one column) or 'nsr' (NSRResult: reward in column 0, novelty in column NOVELTY_COLUMN = 1, ranked by the
MultiObjective blend w r_0 + (1 - w) r_1 with w = ``moo_w``); a capture with an archive and no objective is 'nsr'.

The closed loop (``Capture.obs0`` given: ClosedLoopEnv's obs_0, A^T [band, obs], B^T [act, obs]) has no full-population truth:
  2 obstat      count and n_saved exact; sum and sumsq against the float64 truth's osum / osq of the saved evaluations within
                closed_f64's bound (T ulps of their magnitude per saved evaluation plus OBS_ERR per observation);
  3 normalise   inside the rollout kernel: judged through the fitness;
  4 fitness     closed_f64.truth (with the policy's activation) on a sample (``closed_sample``: every saved evaluation, the first and last pair of each
                stream, random pairs up to about 64 evaluations), with closed_f64's bounds, after closed_f64.growth
                has shown that the sample does not amplify rounding (<= GROWTH_BOUND);
  6 weights     exact against the oracle on the device's fitness; the ranks against the truth are not compared (reported).

Every check is a ``Check``: a measured value, its bound and whether it passed.  Tolerance checks measure a ratio against a
positive bound.  Exact checks measure a distance -- float32 / float64 values in units in the last place of the reference
value, integers in units -- against the bound 0; their margin is the distance itself (1 is the smallest that fails), so a
margin reported for an exact check is an ulp distance, not a multiple of a tolerance.
``assert_ok`` raises a ``StageFailure`` that names every failing stage.
"""
from __future__ import annotations

import math
import os
import sys
from dataclasses import dataclass, field
from typing import List, NamedTuple, Optional, Sequence

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import es_oracle as orc  # noqa: E402
import closed_f64 as cf  # noqa: E402
import f64_rollout as f64  # noqa: E402
import rc_f64 as rc  # noqa: E402
import test_gpu_activations as act_bounds  # noqa: E402
import test_gpu_noise_table as noise_criterion  # noqa: E402
import test_gpu_rollout_f64 as rollout_f64  # noqa: E402

F32 = np.float32
TIE_REL = 1e-12           # the device float64 truth against the CPU float64 reference, relative to the reward mass
# |kappa| of e = kappa f + c + r fitted over a population: the part of the fitness error proportional to the fitness.  Largest
# values measured on an H100 SXM (80 GB, 700 W): ES_ROLLOUT_TC3 8.7e-7 at 376-64-64-17 (rollout_tc2.cu, configs 3, 4 and 5,
# every generation) and 1.33e-6 at the shipped configs' wide policies (rollout_tcw.cu: 1.04e-6 .. 1.33e-6 over simple_conf,
# nsra, ns and flagrun); ES_ROLLOUT_F32 at most 2.7e-8; ES_ROLLOUT_TC (single float16 products, rollout_tcw.cu) 4.1e-5 at
# simple_conf
KAPPA_BOUND = 2.7e-6
KAPPA_BOUND_TC = 8e-5
# the same for the other activations (tests/test_gpu_generation_activations.py), measured there: TC3 3.23e-6 (leaky ReLU at
# obj), 2.51e-6 (ELU at flagrun), 1.99e-6 (ReLU at simple_conf), 1.02e-6 (sigmoid at nsra); F32 at most 7.7e-9 (ReLU at
# 376-64-64-17).  About twice that
KAPPA_BOUND_ACT = 6.5e-6
NOVELTY_COLUMN = 1        # NSRResult's row: [reward, novelty]
GROWTH_BOUND = 100.0      # closed loop: the largest growth of a 1e-9 move of obs_0 over an episode (test_gpu_closed_f64.py)
CLOSED_SAMPLE = 64        # closed loop: evaluations in the fitness truth's sample, at least
STAGES = ('draws', 'obstat', 'normalise', 'fitness', 'novelty', 'weights', 'gradient', 'optimizer')


class Check(NamedTuple):
    stage: str
    name: str
    value: float
    bound: float
    ok: bool
    detail: str = ''

    @property
    def margin(self) -> float:
        """How far the value is from passing: value / bound, or for an exact check (bound 0) the distance itself."""
        return self.value / self.bound if self.bound > 0 else self.value

    def __str__(self):
        return f'[{self.stage}] {self.name}: {self.value:.4g} (bound {self.bound:.4g}){"" if self.ok else "  FAILED"}' + \
               (f'  {self.detail}' if self.detail else '')


class StageFailure(AssertionError):
    def __init__(self, failed: Sequence[Check]):
        self.failed = list(failed)
        self.stages = sorted({c.stage for c in failed}, key=STAGES.index)
        super().__init__('generation stage(s) ' + ', '.join(self.stages) + ' failed:\n' + '\n'.join(map(str, failed)))


@dataclass
class Capture:
    """One generation as captured.  Arrays are numpy except ``table`` (a torch tensor: on the device for the benchmarked
    sizes) and ``act_noise`` (numpy or torch, read one stream's block at a time)."""
    sizes: List[int]
    T: int
    sigma: float
    l2coeff: float
    ob_clip: float
    pos_scale: float
    save_obs_chance: float
    ac_std: float
    lr: float
    table: torch.Tensor
    obs_stream: np.ndarray                  # [T + 1, obs] float32
    rew_vec: np.ndarray                     # [T, act] float32
    # the state at the start
    theta0: np.ndarray
    m0: np.ndarray
    v0: np.ndarray
    t0: int
    streams0: list                          # [(key uint32[624], pos, has_gauss, gauss)] per stream
    ob_mean: np.ndarray
    ob_std: np.ndarray
    # what the generation produced
    idx: np.ndarray                         # int64 [K]
    coin_words: np.ndarray                  # uint32 [K, 4]: (+ evaluation's two words, - evaluation's two words)
    obsn: np.ndarray                        # float32 [T, obs]
    fit: np.ndarray                         # float64 [2, K, n_obj]
    stats: np.ndarray                       # float64 [2 obs + 2]: sum, sumsq, count, n_saved
    weights: np.ndarray                     # float32 [K]
    n_ranked: int
    gsum: np.ndarray                        # float32 [P]
    theta1: np.ndarray
    m1: np.ndarray
    v1: np.ndarray
    t1: int
    streams1: list                          # the streams after the generation
    behv: Optional[np.ndarray] = None       # float32 [2, K, 3]
    act_noise: object = None                # float32 [K, 2, E * T * act], the episodes back to back
    archive: Optional[np.ndarray] = None    # float64 [A, 2]
    nov_k: int = 10
    moo_w: float = 0.5                      # 'nsr': the weight of the reward column's ranks (the novelty's: 1 - moo_w)
    beta1: float = 0.9
    beta2: float = 0.999
    epsilon: float = 1e-08
    episodes: int = 1
    objective: Optional[str] = None         # 'reward' or 'nsr' (novelty in column NOVELTY_COLUMN); None: 'nsr' with an archive
    # the closed loop (ClosedLoopEnv.device_closed): obs_0 [obs], A^T [band, obs], B^T [act, obs]; obs_stream and obsn unused
    obs0: Optional[np.ndarray] = None
    env_a: Optional[np.ndarray] = None
    env_b: Optional[np.ndarray] = None
    band: Optional[int] = None
    # the policy's activation after every layer (an nn.Activation; None: tanh), applied by every float64 truth
    activation: object = None
    extra: dict = field(default_factory=dict)

    def __post_init__(self):
        if self.objective is None:
            self.objective = 'reward' if self.archive is None else 'nsr'
        assert self.objective in ('reward', 'nsr') and (self.objective == 'nsr') == (self.archive is not None)

    @property
    def closed(self) -> bool:
        return self.obs0 is not None

    @property
    def obs_dim(self) -> int:
        return self.sizes[0]

    @property
    def P(self) -> int:
        return f64.n_params(self.sizes)

    @property
    def K(self) -> int:
        return len(self.idx)

    @property
    def n_per_stream(self) -> int:
        return self.K // len(self.streams0)

    @property
    def act(self) -> int:
        return self.sizes[-1]


# ---------------------------------------------------------------------------------------------- distances
def ulps(got, want) -> float:
    """Largest |got - want| in units in the last place of ``want`` (its own float dtype); integers: in units."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        return math.inf
    if want.dtype.kind in 'iub':
        return float(np.abs(got.astype(np.float64) - want.astype(np.float64)).max(initial=0.0))
    if np.isnan(got).any() or np.isnan(want).any():
        return 0.0 if np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)]) \
            else math.inf
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    sp = np.spacing(np.abs(want).astype(want.dtype)).astype(np.float64)
    return float((d / sp).max(initial=0.0))


def _exact(stage, name, got, want, detail=''):
    u = ulps(got, want)
    return Check(stage, name, u, 0.0, u == 0, detail)


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


# ---------------------------------------------------------------------------------------------- 1. draws
def replay_stream(cap: Capture, r: int):
    """Stream r in the reference's order.  Returns (indices, coin words [n, 4] uint32, end state, the noise block
    [n, 2, E T act] float64 (ac_std * randn, the E episodes of an evaluation back to back) or None)."""
    key, pos, has, gauss = cap.streams0[r]
    rs = np.random.RandomState()
    rs.set_state(('MT19937', np.asarray(key, dtype=np.uint32), int(pos), int(has), float(gauss)))
    n, L, P = cap.n_per_stream, cap.table.numel(), cap.P
    nrm = cap.episodes * cap.T * cap.act if cap.ac_std else 0
    idx = np.empty(n, dtype=np.int64)
    words = np.empty((n, 4), dtype=np.uint32)
    noise = np.empty((n, 2, nrm), dtype=np.float64) if nrm else None
    for k in range(n):
        idx[k] = orc.sample_idx(L, rs, P)
        for s in range(2):
            # fit_fn's rs.random() (simple_example.py:38): two raw 32-bit words
            words[k, 2 * s] = int.from_bytes(rs.bytes(4), 'little')
            words[k, 2 * s + 1] = int.from_bytes(rs.bytes(4), 'little')
            if nrm:
                noise[k, s] = rs.randn(nrm) * cap.ac_std          # per episode FeedForward.forward's T x rs.randn(act) * ac_std
    return idx, words, rs.get_state(), noise


def saved_flags(words: np.ndarray, chance: float) -> np.ndarray:
    """[..., 4] coin words -> [..., 2] save_obs flags (rs.random() < chance)."""
    w = words.astype(np.uint64).reshape(-1, 2, 2)
    u = ((w[..., 0] >> np.uint64(5)).astype(np.float64) * 67108864.0 + (w[..., 1] >> np.uint64(6)).astype(np.float64)) \
        / 9007199254740992.0
    return (u < chance).reshape(words.shape[:-1] + (2,))


def stage_draws(cap: Capture) -> List[Check]:
    """Leaves the replayed coin words of every stream in ``cap.extra['replay_words']`` (stage 2 counts the saves from them)."""
    out = []
    n = cap.n_per_stream
    bad_idx = bad_words = bad_state = 0.0
    noise_mism = 0
    noise_fail = ''
    cap.extra['replay_words'] = []
    for r in range(len(cap.streams0)):
        idx, words, st, noise = replay_stream(cap, r)
        cap.extra['replay_words'].append(words)
        sl = slice(r * n, (r + 1) * n)
        bad_idx = max(bad_idx, ulps(cap.idx[sl], idx))
        bad_words = max(bad_words, ulps(cap.coin_words[sl], words))
        key1, pos1, has1, gauss1 = cap.streams1[r]
        bad_state = max(bad_state, ulps(np.asarray(key1, dtype=np.uint32), st[1]), abs(int(pos1) - st[2]), abs(int(has1) - st[3]))
        g = abs(float(gauss1) - st[4]) / np.spacing(abs(st[4])) if st[4] != 0 else abs(float(gauss1)) * math.inf
        if g > 2:
            bad_state = max(bad_state, g)
        if cap.ac_std:
            got = _np(cap.act_noise[sl])
            try:
                noise_mism += noise_criterion._mismatches(got.reshape(-1), noise.reshape(-1))
            except AssertionError as ex:
                noise_fail = f'stream {r}: ' + str(ex)[:200]
    out.append(Check('draws', 'noise indices (units)', bad_idx, 0.0, bad_idx == 0))
    out.append(Check('draws', 'coin words (units)', bad_words, 0.0, bad_words == 0))
    out.append(Check('draws', 'end states: key / pos / has_gauss (units), cached gaussian beyond 2 ulp', bad_state, 0.0,
                     bad_state == 0))
    if cap.ac_std:
        out.append(Check('draws', 'action noise outside the midpoint criterion', 0.0 if not noise_fail else 1.0, 0.0,
                         not noise_fail, f'{noise_mism} values one ulp away next to a midpoint' + (f'; {noise_fail}' if noise_fail else '')))
        cap.extra['noise_1ulp'] = noise_mism
    return out


# ---------------------------------------------------------------------------------------------- 2. obstat
def _replay_words(cap: Capture) -> list:
    if 'replay_words' not in cap.extra:
        cap.extra['replay_words'] = [replay_stream(cap, r)[1] for r in range(len(cap.streams0))]
    return cap.extra['replay_words']


def replayed_saves(cap: Capture) -> np.ndarray:
    """[2, K] bool: the evaluations whose replayed save_obs coin fell."""
    return np.concatenate([saved_flags(w, cap.save_obs_chance) for w in _replay_words(cap)]).T.copy()


def stage_obstat(cap: Capture, truth=None) -> List[Check]:
    if cap.closed:
        return _stage_obstat_closed(cap, truth)
    obs = cap.obs_stream.shape[1]
    flags = np.concatenate([saved_flags(replay_words, cap.save_obs_chance) for replay_words in cap.extra['replay_words']])
    s, q, c = orc.ob_sum_sq_cnt(cap.obs_stream[1:cap.T + 1])
    st = orc.ObStatOracle((obs,), 0)
    zeros = np.zeros(obs)
    for saved in flags.reshape(-1):                          # evaluation order: stream, pair, + then -
        if saved:
            st.inc(s, q, c)
        else:
            st.inc(zeros, zeros, 0)
    n_saved = int(flags.sum())
    cap.extra['n_saved'] = n_saved
    return [_exact('obstat', 'sum (ulp)', cap.stats[:obs], st.sum),
            _exact('obstat', 'sumsq (ulp)', cap.stats[obs:2 * obs], st.sumsq),
            _exact('obstat', 'count (ulp)', cap.stats[2 * obs:2 * obs + 1], np.array([float(st.count)])),
            _exact('obstat', 'n_saved (units)', cap.stats[2 * obs + 1:], np.array([float(n_saved)]), f'{n_saved} saves')]


def _truth_columns(truth, saved: np.ndarray):
    """The sampled truth's [2, n] positions of the saved evaluations ([2, K] mask); raises when the sample misses one."""
    col = {p: j for j, p in enumerate(truth['pairs'])}
    s_idx, k_idx = np.nonzero(saved)
    missing = sorted({int(k) for k in k_idx if int(k) not in col})
    if missing:
        raise ValueError(f'saved evaluations of pairs {missing[:8]} are not in the truth sample')
    return s_idx, np.array([col[int(k)] for k in k_idx], dtype=np.int64)


def _stage_obstat_closed(cap: Capture, truth) -> List[Check]:
    """Every evaluation's ObStat increment is its own post-step observations (obs_1 .. obs_T of the last episode): count and
    n_saved exact, the sums within closed_f64's bound of the truth's (the device adds them with float64 atomics,
    in no fixed order)."""
    obs, T = cap.obs_dim, cap.T
    saved = replayed_saves(cap)
    n_saved = int(saved.sum())
    cap.extra['n_saved'] = n_saved
    s_idx, j_idx = _truth_columns(truth, saved)
    U, ns = 2.0 ** -24, max(1, n_saved)
    want_s = truth['osum'][s_idx, j_idx].sum(axis=0)
    want_q = truth['osq'][s_idx, j_idx].sum(axis=0)
    bound_s = 2 * T * U * truth['oabs'][s_idx, j_idx].sum(axis=0) + cf.OBS_ERR * T * ns
    bound_q = 2 * T * U * want_q + 2 * cf.OBS_ERR * T * ns
    rs = float((np.abs(cap.stats[:obs] - want_s) / bound_s).max())
    rq = float((np.abs(cap.stats[obs:2 * obs] - want_q) / bound_q).max())
    return [Check('obstat', 'sum err/bound against the float64 truth', rs, 1.0, rs <= 1.0),
            Check('obstat', 'sumsq err/bound against the float64 truth', rq, 1.0, rq <= 1.0),
            _exact('obstat', 'count (ulp)', cap.stats[2 * obs:2 * obs + 1], np.array([float(T * n_saved)])),
            _exact('obstat', 'n_saved (units)', cap.stats[2 * obs + 1:], np.array([float(n_saved)]), f'{n_saved} saves')]


# ---------------------------------------------------------------------------------------------- 3. normalise
def stage_normalise(cap: Capture) -> List[Check]:
    if cap.closed:
        return []                                         # the closed-loop kernel normalises every step itself
    want = orc.normalise_obs(cap.obs_stream[:cap.T], cap.ob_mean, cap.ob_std, cap.ob_clip)
    return [_exact('normalise', 'obsn (ulp)', cap.obsn, want)]


# ---------------------------------------------------------------------------------------------- 4. fitness
ACT_BYTES = 2 ** 29       # fitness_truth: the float64 activations of one layer held per chunk of pairs, at most


def layer_forms(cap: Capture, xp=np) -> list:
    """The float64 activation of every layer of ``cap``'s policy (f64_rollout.form of ``cap.activation``; tanh for None), for
    numpy arrays or (``xp=torch``) torch tensors."""
    return [f64.form(cap.activation, xp)] * (len(cap.sizes) - 1)


def fitness_truth(cap: Capture, chunk: Optional[int] = None, behaviour_episode: int = -1, noise=None, acts=None):
    """(fitness [2, K], behaviour [2, K, 3], reward mass [2, K], position magnitude [2, K, 3]) in float64 (f64_rollout's
    definitions, with the policy's activation in its forms), computed with torch.float64 on the table's device in
    chunks of pairs: a measurement reference.  The forward pass is shared by the E episodes (only the noise differs); fitness
    and mass are the per-step means over them, behaviour and magnitude the episode ``behaviour_episode``'s.  ``chunk``
    (default: up to 200 pairs, fewer where one layer's activations over T steps would pass ACT_BYTES); ``noise``: in place of
    ``cap.act_noise``; ``acts``: torch functions, one per layer, in place of ``layer_forms(cap, torch)``."""
    dev = cap.table.device
    d64 = torch.float64
    sizes, T, act, K, P, E = cap.sizes, cap.T, cap.act, cap.K, cap.P, cap.episodes
    if chunk is None:
        chunk = max(1, min(200, ACT_BYTES // (8 * T * max(sizes[1:]))))
    noise = cap.act_noise if noise is None else noise
    theta = torch.from_numpy(np.ascontiguousarray(cap.theta0)).to(dev, d64)
    X = torch.from_numpy(np.ascontiguousarray(cap.obsn)).to(dev, d64)
    C = torch.from_numpy(np.ascontiguousarray(cap.rew_vec)).to(dev, d64)
    idx_all = torch.from_numpy(np.ascontiguousarray(cap.idx)).to(dev)
    ar = torch.arange(P, device=dev)
    s32 = float(np.float32(cap.sigma))
    ps = float(cap.pos_scale)
    lay = f64.layer_slices(sizes)
    acts = layer_forms(cap, torch) if acts is None else list(acts)
    sel = [j % act for j in range(3)]
    fit, mass = np.zeros((2, K)), np.zeros((2, K))
    behv, mag = np.zeros((2, K, 3)), np.zeros((2, K, 3))
    for b0 in range(0, K, chunk):
        b1 = min(K, b0 + chunk)
        eps = cap.table[idx_all[b0:b1, None] + ar[None, :]].to(d64)
        nz_block = None if not cap.ac_std else torch.as_tensor(_np(noise[b0:b1])).to(dev, d64)
        for s, sign in enumerate((1.0, -1.0)):
            W = theta[None, :] + sign * s32 * eps                                 # [B, P]
            B = W.shape[0]
            wo, bo, fi, fo = lay[0]
            W1 = W[:, wo:wo + fi * fo].reshape(B, fo, fi)
            a = acts[0]((X @ W1.reshape(B * fo, fi).T).reshape(T, B, fo).permute(1, 0, 2) + W[:, bo:bo + fo][:, None, :])
            for (wo, bo, fi, fo), act_fn in zip(lay[1:], acts[1:]):
                a = act_fn(torch.bmm(a, W[:, wo:wo + fi * fo].reshape(B, fo, fi).transpose(1, 2)) + W[:, bo:bo + fo][:, None, :])
            if nz_block is None:
                prod = a * C[None]
                fit[s, b0:b1] = prod.sum(dim=(1, 2)).cpu().numpy()
                mass[s, b0:b1] = prod.abs().sum(dim=(1, 2)).cpu().numpy()
                ab = a
            else:
                nz_e = nz_block[:, s].reshape(B, E, T, act)
                f_acc = torch.zeros(B, dtype=d64, device=dev)
                m_acc = torch.zeros(B, dtype=d64, device=dev)
                for e in range(E):
                    prod = (a + nz_e[:, e]) * C[None]
                    f_acc += prod.sum(dim=(1, 2))
                    m_acc += prod.abs().sum(dim=(1, 2))
                fit[s, b0:b1] = (f_acc / E).cpu().numpy()
                mass[s, b0:b1] = (m_acc / E).cpu().numpy()
                ab = a + nz_e[:, behaviour_episode]
            terms = ps * ab[:, :, sel]
            behv[s, b0:b1] = terms.sum(dim=1).cpu().numpy()
            mag[s, b0:b1] = (torch.cumsum(terms, dim=1).abs().sum(dim=1) + terms.abs().sum(dim=1)).cpu().numpy()
    return fit, behv, mass, mag


def tie_pairs(cap: Capture) -> List[int]:
    """The first and last pair of every stream (>= 16 evaluations with 4 streams or more)."""
    n = cap.n_per_stream
    return sorted({p for r in range(len(cap.streams0)) for p in (r * n, r * n + n - 1)})


def closed_sample(cap: Capture, seed: int = 0) -> List[int]:
    """The pairs the closed-loop truth covers: every pair with a saved evaluation (the replayed coins), the first and last
    pair of every stream, then random pairs until the sample holds CLOSED_SAMPLE evaluations."""
    saved = replayed_saves(cap)
    pairs = set(np.nonzero(saved.any(axis=0))[0].tolist()) | set(tie_pairs(cap))
    for p in np.random.RandomState(seed).permutation(cap.K):
        if 2 * len(pairs) >= CLOSED_SAMPLE:
            break
        pairs.add(int(p))
    return sorted(pairs)


def closed_truth(cap: Capture, pairs: Optional[Sequence[int]] = None, growth: bool = True, acts=None):
    """closed_f64.truth of the pairs ``pairs`` (default closed_sample) from the device's indices, theta, observation
    statistics and action noise, with the policy's activation (``layer_forms(cap)``, or ``acts``: numpy functions, one per
    layer), plus 'pairs' and 'growth' (closed_f64.growth of the same evaluations; nan when not ``growth``)."""
    pairs = closed_sample(cap) if pairs is None else list(pairs)
    P = cap.P
    table_np = np.concatenate([_np(cap.table[int(cap.idx[k]):int(cap.idx[k]) + P]) for k in pairs])
    noise = None
    if cap.ac_std:
        noise = np.stack([_np(cap.act_noise[k]) for k in pairs])
    args = (table_np, np.arange(len(pairs)) * P, cap.theta0, cap.sigma, cap.sizes, cap.ob_mean, cap.ob_std, cap.ob_clip,
            cap.obs0, cap.env_a, cap.env_b, cap.rew_vec, cap.pos_scale)
    kw = dict(act_noise=noise, episodes=cap.episodes if cap.ac_std else 1,
              activation=layer_forms(cap) if acts is None else list(acts))
    out = cf.truth(*args, **kw)
    out['growth'] = cf.growth(*args, **kw) if growth else math.nan
    out['pairs'] = pairs
    return out


def _stage_fitness_closed(cap: Capture, truth) -> List[Check]:
    """The sampled evaluations against the float64 truth, with closed_f64's bounds (test_gpu_closed_f64._check's)."""
    pairs = truth['pairs']
    U = 2.0 ** -24
    f = cap.fit[:, pairs, 0]
    tf, mass = truth['fit'], truth['mass']
    err = np.abs(f - tf)
    spread = max(tf.std(), 1e-3 * math.sqrt(cap.T))
    rms = math.sqrt((err ** 2).mean())
    worst = float((err / mass).max())
    g = truth['growth']
    out = [Check('fitness', 'closed loop: growth of a 1e-9 move of obs_0 (the sample is not chaotic)', g, GROWTH_BOUND,
                 g <= GROWTH_BOUND, f'{2 * len(pairs)} evaluations sampled'),
           Check('fitness', 'max err/mass', worst, cf.EVAL_REL, worst <= cf.EVAL_REL),
           Check('fitness', 'rms/spread', rms / spread, cf.RMS_BOUND, rms <= cf.RMS_BOUND * spread)]
    if cap.behv is not None:
        tol = 2 * U * truth['mag'] + cf.ACT_ERR * float(np.float32(cap.pos_scale)) * cap.T
        r = float((np.abs(cap.behv[:, pairs] - truth['behv']) / tol).max())
        out.append(Check('fitness', 'behaviour err/tol', r, 1.0, r <= 1.0))
    cap.extra['fitness'] = dict(sampled_evaluations=2 * len(pairs), rms_over_spread=rms / spread, max_err_over_mass=worst,
                                growth=g)
    return out


def stage_fitness(cap: Capture, mode: int, truth, tie: Optional[Sequence[int]] = None) -> List[Check]:
    if cap.closed:
        return _stage_fitness_closed(cap, truth)
    tf, tb, mass, mag = truth
    f = cap.fit[:, :, 0]
    b = cap.behv
    case = type('Case', (), dict(T=cap.T, ps=cap.pos_scale))()
    err = np.abs(f - tf)
    spread = max(tf.std(), 1e-3 * math.sqrt(cap.T))
    rms = math.sqrt((err ** 2).mean())
    worst = float((err / mass).max())
    # the rms bound of the policy's activation: test_gpu_rollout_f64's for tanh, test_gpu_activations' for the others
    rms_bound = rollout_f64.RMS_BOUND[mode] if cap.activation is None else act_bounds.rms_bound(mode, cap.activation)
    out = [Check('fitness', 'max err/mass', worst, rollout_f64.EVAL_REL[mode], worst <= rollout_f64.EVAL_REL[mode]),
           Check('fitness', 'rms/spread', rms / spread, rms_bound, rms <= rms_bound * spread)]
    if b is not None:
        tol = 2 * rollout_f64.U * mag + rollout_f64.ACT_ERR[mode] * cap.pos_scale * cap.T
        r = float((np.abs(b - tb) / tol).max())
        out.append(Check('fitness', 'behaviour err/tol', r, 1.0, r <= 1.0))
    # the error's part proportional to the fitness, fitted over the population (e = kappa f + c + r), and the rms of what remains:
    # a positive rescaling and a common offset leave every rank unchanged, so they are reported apart from the residual
    A = np.stack([tf.reshape(-1), np.ones(tf.size)], 1)
    coef = np.linalg.lstsq(A, (f - tf).reshape(-1), rcond=None)[0]
    kappa, resid = coef[0], (f - tf).reshape(-1) - A @ coef
    cap.extra['fitness'] = dict(rms_over_spread=rms / spread, mean_err=float((f - tf).mean()), mean_fitness=float(tf.mean()),
                                kappa=float(kappa), resid_rms_over_spread=float(math.sqrt((resid ** 2).mean()) / spread))
    out.append(Check('fitness', 'rms/spread of the error less its fitted scale and offset',
                     cap.extra['fitness']['resid_rms_over_spread'], rms_bound,
                     cap.extra['fitness']['resid_rms_over_spread'] <= rms_bound))
    kb = KAPPA_BOUND_TC if mode == rollout_f64.TC else KAPPA_BOUND if cap.activation is None else KAPPA_BOUND_ACT
    out.append(Check('fitness', '|fitted relative scale of the error|', abs(float(kappa)), kb, abs(float(kappa)) <= kb))
    if cap.activation is None:                             # the one assert helper of the tanh rollout tests decides as well
        try:
            rollout_f64._check('generation', mode, case, f, b, None, truth)
            helper_ok = True
        except AssertionError:
            helper_ok = False
        if helper_ok != all(c.ok for c in out[:3 if b is not None else 2]):
            out.append(Check('fitness', 'test_gpu_rollout_f64._check disagrees', 1.0, 0.0, False))
    # the device float64 truth against the plain CPU reference on sampled pairs
    tie = tie_pairs(cap) if tie is None else list(tie)
    P = cap.P
    table_np = np.concatenate([_np(cap.table[int(cap.idx[k]):int(cap.idx[k]) + P]) for k in tie])
    noise = None
    if cap.ac_std:
        noise = np.stack([_np(cap.act_noise[k]) for k in tie])
    tie_args = (table_np, np.arange(len(tie)) * P, cap.theta0, cap.sigma, cap.sizes, cap.obsn, cap.rew_vec, cap.pos_scale)
    rf, rb, rm, rmag = f64.rollout_f64(*tie_args, noise, cap.episodes, activation=f64.form(cap.activation))
    rel = float(max((np.abs(rf - tf[:, tie]) / rm).max(), (np.abs(rb - tb[:, tie]) / np.maximum(rmag, 1e-300)).max()))
    out.append(Check('fitness', f'float64 truth vs CPU reference ({2 * len(tie)} evaluations), rel', rel, TIE_REL, rel <= TIE_REL))
    return out


# ---------------------------------------------------------------------------------------------- 5. novelty
def stage_novelty(cap: Capture) -> List[Check]:
    if cap.archive is None:
        return []
    b = cap.behv
    want = np.array([[orc.novelty(b[s, k, :2], cap.archive, cap.nov_k) for k in range(cap.K)] for s in range(2)])
    return [_exact('novelty', f'novelty column {NOVELTY_COLUMN} (ulp)', cap.fit[:, :, NOVELTY_COLUMN], want,
                   f'archive of {len(cap.archive)}, k = {cap.nov_k}')]


# ---------------------------------------------------------------------------------------------- 6. weights
def reference_weights(cap: Capture, fit: np.ndarray, moo_w: Optional[float] = None):
    """Centered ranks of the reward, or for 'nsr' the MultiObjective blend of the reward's (weight ``moo_w``, default the
    capture's) and the novelty's ranks."""
    if cap.objective == 'reward':
        w, n = orc.centered_ranker(fit[0][:, :1], fit[1][:, :1])
    else:
        cols = [0, NOVELTY_COLUMN]
        w, n = orc.moo_ranker(fit[0][:, cols], fit[1][:, cols], cap.moo_w if moo_w is None else moo_w)
    return np.asarray(w, dtype=F32).reshape(-1), n


def rank_report(cap: Capture, truth_fit: np.ndarray):
    """Against the float64 truth's ranks (column 0; with an archive the device's novelty is the truth's second column):
    (ranks differing, largest rank shift, largest |dw|)."""
    f = cap.fit[:, :, 0].reshape(-1)
    t = truth_fit.reshape(-1)
    dr = np.abs(orc.rank(f) - orc.rank(t))
    tfit = cap.fit.copy()
    tfit[:, :, 0] = truth_fit
    wt, _ = reference_weights(cap, tfit)
    return int((dr != 0).sum()), int(dr.max()), float(np.abs(cap.weights.astype(np.float64) - wt).max())


def stage_weights(cap: Capture, truth_fit=None, shift_bound=None, dw_bound=None) -> List[Check]:
    w, n = reference_weights(cap, cap.fit)
    out = [_exact('weights', 'weights (ulp)', cap.weights, w),
           Check('weights', 'n_ranked (units)', float(abs(cap.n_ranked - n)), 0.0, cap.n_ranked == n)]
    if cap.closed:
        cap.extra['ranks_vs_truth'] = 'not compared: the closed loop has a float64 truth of a sample only'
        out.append(Check('weights', 'ranks against the float64 truth: not compared (closed loop, sampled truth)', 0.0, 0.0,
                         True))
    elif truth_fit is not None:
        nd, shift, dw = rank_report(cap, truth_fit)
        cap.extra['ranks_vs_truth'] = dict(ranks_differing=nd, max_rank_shift=shift, max_abs_dw=dw)
        out.append(Check('weights', 'largest rank shift against the float64 truth', shift, shift_bound, shift <= shift_bound,
                         f'{nd} of {2 * cap.K} ranks differ'))
        out.append(Check('weights', 'largest |dw| against the float64 truth', dw, dw_bound, dw <= dw_bound))
    return out


# ---------------------------------------------------------------------------------------------- 7. gradient
def stage_gradient(cap: Capture, sm: int) -> List[Check]:
    dev = cap.table.device
    idx = torch.from_numpy(np.ascontiguousarray(cap.idx)).to(dev)
    w = torch.from_numpy(np.ascontiguousarray(cap.weights)).to(dev)
    truth, mass = rc.truth_device(cap.table, idx, w, cap.P)
    worst, rms = rc.judge(cap.gsum, truth.cpu().numpy(), mass.cpu().numpy(), rc.rc_layout(cap.P, cap.K, sm))
    return [Check('gradient', 'rc worst (of its per-column bound)', worst, 1.0, worst <= 1.0),
            Check('gradient', 'rc rms (U M_p)', rms, rc.RMS_BOUND, rms <= rc.RMS_BOUND)]


# ---------------------------------------------------------------------------------------------- 8. optimizer
def adam_reference(cap: Capture, n_ranked: int):
    """es.approx_grad's update in float32 (es.py:100-101, policy.py:73-74) on the device's gsum and theta."""
    opt = orc.AdamOracle(cap.P, cap.lr, cap.beta1, cap.beta2, cap.epsilon)
    opt.m, opt.v, opt.t = cap.m0.astype(F32).copy(), cap.v0.astype(F32).copy(), int(cap.t0)
    flat = cap.theta0.astype(F32).copy()
    grad = (cap.gsum.astype(F32) / F32(n_ranked)).astype(F32)
    g = ((F32(cap.l2coeff) * flat).astype(F32) - grad).astype(F32)
    flat += opt.step(g)
    return flat, opt.m, opt.v, opt.t


def stage_optimizer(cap: Capture) -> List[Check]:
    _, n = reference_weights(cap, cap.fit)
    th, m, v, t = adam_reference(cap, n)
    return [_exact('optimizer', 'theta (ulp)', cap.theta1, th), _exact('optimizer', 'm (ulp)', cap.m1, m),
            _exact('optimizer', 'v (ulp)', cap.v1, v), Check('optimizer', 't (units)', abs(cap.t1 - t), 0.0, cap.t1 == t)]


# ---------------------------------------------------------------------------------------------- all stages
def judge(cap: Capture, mode: int, sm: int, shift_bound: float, dw_bound: float, truth=None,
          tie: Optional[Sequence[int]] = None) -> List[Check]:
    """Every stage of ``cap``, in order; a stage that raises counts as failed.  ``truth``: fitness_truth(cap) (closed loop:
    closed_truth(cap)) when already computed (re-judging mutated copies of a large capture whose mutation leaves the rollout
    inputs alone)."""
    if truth is None and not cap.closed:
        truth = fitness_truth(cap)
    held = [truth]

    def tr():                   # the closed loop's sample holds the saved evaluations: computed after the draws' replay
        if held[0] is None:
            held[0] = cap.extra['closed_truth'] = closed_truth(cap)
        return held[0]
    checks = []
    for stage, fn in (('draws', lambda: stage_draws(cap)), ('obstat', lambda: stage_obstat(cap, tr() if cap.closed else None)),
                      ('normalise', lambda: stage_normalise(cap)), ('fitness', lambda: stage_fitness(cap, mode, tr(), tie)),
                      ('novelty', lambda: stage_novelty(cap)),
                      ('weights', lambda: stage_weights(cap, None if cap.closed else tr()[0], shift_bound, dw_bound)),
                      ('gradient', lambda: stage_gradient(cap, sm)), ('optimizer', lambda: stage_optimizer(cap))):
        try:
            checks += fn()
        except Exception as ex:                                    # noqa: BLE001 -- reported as the stage's failure
            checks.append(Check(stage, f'raised {type(ex).__name__}', math.inf, 0.0, False, str(ex)[:300]))
    return checks


def failed(checks: Sequence[Check]) -> List[Check]:
    return [c for c in checks if not c.ok]


def assert_ok(checks: Sequence[Check]):
    bad = failed(checks)
    if bad:
        raise StageFailure(bad)


def report(title: str, checks: Sequence[Check]) -> str:
    return '\n'.join([f'== {title}'] + [f'  {c}' for c in checks])


# ---------------------------------------------------------------------------------------------- modelled pipeline bugs
def _copy(cap: Capture, **changes) -> Capture:
    import copy
    out = copy.copy(cap)
    out.extra = {}
    for k, v in changes.items():
        setattr(out, k, v)
    return out


def _block(a, r, n):
    return slice(r * n, (r + 1) * n)


def _stats_with(cap: Capture, n_saved: int, obs_stream: np.ndarray) -> np.ndarray:
    """The generation statistics of ``n_saved`` saves of ``obs_stream``'s post-step rows, summed in order."""
    obs = cap.obs_stream.shape[1]
    s, q, c = orc.ob_sum_sq_cnt(obs_stream[1:cap.T + 1])
    st = orc.ObStatOracle((obs,), 0)
    for _ in range(n_saved):
        st.inc(s, q, c)
    return np.concatenate([st.sum, st.sumsq, [float(st.count), float(n_saved)]])


def _n_saved(cap: Capture) -> int:
    return int(cap.stats[2 * cap.obs_stream.shape[1] + 1])


def _optimizer_after(cap: Capture, n_ranked=None, l2coeff=None, t0=None):
    c = _copy(cap, l2coeff=cap.l2coeff if l2coeff is None else l2coeff, t0=cap.t0 if t0 is None else t0)
    th, m, v, _ = adam_reference(c, reference_weights(cap, cap.fit)[1] if n_ranked is None else n_ranked)
    return dict(theta1=th, m1=m, v1=v)


def _gsum_of(cap: Capture, idx: np.ndarray, w: np.ndarray) -> np.ndarray:
    """sum_k w_k eps_idx_k, rounded once to float32 (a correct reconstruction of the given pairing)."""
    dev = cap.table.device
    t, _ = rc.truth_device(cap.table, torch.from_numpy(np.ascontiguousarray(idx)).to(dev),
                           torch.from_numpy(np.ascontiguousarray(w)).to(dev), cap.P)
    return t.cpu().numpy().astype(F32)


def _m_shift_stream(c):
    n = c.n_per_stream
    idx = c.idx.copy()
    idx[_block(idx, 1, n)] = np.roll(idx[_block(idx, 1, n)], -1)       # stream 1 writes pair k + 1's index into slot k
    return _copy(c, idx=idx)


def _m_swap_streams(c):
    n, R = c.n_per_stream, len(c.streams0)
    a, b = _block(None, 0, n), _block(None, R - 1, n)
    ch = {}
    for name, axis in (('idx', 0), ('coin_words', 0), ('fit', 1), ('behv', 1), ('weights', 0)):
        x = getattr(c, name)
        if x is None:
            continue
        x = x.copy()
        if axis == 0:
            x[a], x[b] = x[b].copy(), x[a].copy()
        else:
            x[:, a], x[:, b] = x[:, b].copy(), x[:, a].copy()
        ch[name] = x
    return _copy(c, **ch)


def _m_coin_to_neg(c):
    w = c.coin_words.copy()
    w[:, 2:4] = w[:, 0:2]
    return _copy(c, coin_words=w)


def _m_drop_save(c):
    return _copy(c, stats=_stats_with(c, _n_saved(c) - 1, c.obs_stream))


def _m_sign_swap(c):
    f = c.fit.copy()
    k = c.K // 2
    f[:, k] = f[::-1, k].copy()
    return _copy(c, fit=f)


def _m_novelty_column(c):
    return _copy(c, fit=c.fit[:, :, ::-1].copy())


def _m_novelty_off_by_one(c):
    f = c.fit.copy()
    f[:, :, 1] = np.roll(f[:, :, 1].reshape(-1), -1).reshape(2, c.K)
    return _copy(c, fit=f)


def _m_weights_next(c):
    g = _gsum_of(c, np.roll(c.idx, -1), c.weights)                      # w_k paired with idx[k + 1]
    c2 = _copy(c, gsum=g)
    return _copy(c2, **_optimizer_after(c2))


def _m_gsum_over_k(c):
    return _copy(c, **_optimizer_after(c, n_ranked=c.K))


def _m_l2_sign(c):
    return _copy(c, **_optimizer_after(c, l2coeff=-c.l2coeff))


def _m_adam_t(c):
    return _copy(c, t1=c.t0, **_optimizer_after(c, t0=c.t0 - 1))


def _m_std_squared(c):
    return _copy(c, obsn=orc.normalise_obs(c.obs_stream[:c.T], c.ob_mean, np.square(c.ob_std), c.ob_clip))


def _m_stale_colsum(c):
    old = np.random.RandomState(12).randn(*c.obs_stream.shape).astype(F32)    # the stream's content before it was rewritten
    return _copy(c, stats=_stats_with(c, _n_saved(c), old))


def _rescored(c: Capture, moo_w: Optional[float] = None) -> Capture:
    """``c`` with everything after the fitness recomputed correctly from its (mutated) fitness rows: weights, n_ranked,
    gsum and the Adam step -- so that a modelled bug upstream is rejected by the stage it sits in, not by a mismatch it
    leaves downstream."""
    w, n = reference_weights(c, c.fit, moo_w)
    c2 = _copy(c, weights=w, n_ranked=n, gsum=_gsum_of(c, c.idx, w))
    return _copy(c2, **_optimizer_after(c2, n_ranked=n))


def _m_ep0_noise(c):
    nz = _np(c.act_noise).reshape(c.K, 2, c.episodes, -1).copy()
    nz[:, :, 1:] = nz[:, :, :1]
    tf, tb, _, _ = fitness_truth(c, noise=nz.reshape(c.K, 2, -1))
    f = c.fit.copy()
    f[:, :, 0] = tf
    return _rescored(_copy(c, fit=f, behv=None if c.behv is None else tb.astype(F32)))


def _m_episodes_not_divided(c):
    f = c.fit.copy()
    f[:, :, 0] *= c.episodes
    return _rescored(_copy(c, fit=f))


def _m_first_episode_behaviour(c):
    _, tb, _, _ = fitness_truth(c, behaviour_episode=0)
    return _copy(c, behv=tb.astype(F32))


def _m_novelty_over_reward(c):
    f = np.zeros_like(c.fit)                                            # column 1 never written (the buffer's zeros)
    f[:, :, 0] = c.fit[:, :, NOVELTY_COLUMN]
    return _rescored(_copy(c, fit=f))


def _m_moo_w_swapped(c):
    return _rescored(c, moo_w=1 - c.moo_w)                              # w r_novelty + (1 - w) r_reward


def _m_archive_clipped(c):
    """sum of the min(k, A) smallest distances over k."""
    f = c.fit.copy()
    a = np.asarray(c.archive, np.float64)
    for s in range(2):
        for k in range(c.K):
            d = np.sqrt(((a - c.behv[s, k, :2].astype(np.float64)[None, :]) ** 2).sum(axis=1))
            f[s, k, NOVELTY_COLUMN] = float(np.sort(d)[:c.nov_k].sum() / c.nov_k)
    return _rescored(_copy(c, fit=f))


def _closed_saved_sums(c, shift: str = None, drop: int = 0):
    """Closed loop: the statistics of the saved evaluations from the float64 truth, computed wrongly on purpose:
    ``shift`` 'pre' sums obs_0 .. obs_{T-1}, 'short' obs_1 .. obs_{T-1} with T - 1 rows each; ``drop`` leaves out that many
    saved evaluations (the last ones)."""
    truth = c.extra.get('closed_truth') or closed_truth(c, growth=False)
    saved = replayed_saves(c)
    s_idx, j_idx = _truth_columns(truth, saved)
    if drop:
        s_idx, j_idx = s_idx[:-drop], j_idx[:-drop]
    osum, osq = truth['osum'][s_idx, j_idx], truth['osq'][s_idx, j_idx]
    last = truth['olast'][s_idx, j_idx]
    rows = c.T
    o0 = np.asarray(c.obs0, np.float64)[None, :]
    if shift == 'pre':
        osum, osq = osum - last + o0, osq - last ** 2 + o0 ** 2
    elif shift == 'short':
        osum, osq, rows = osum - last, osq - last ** 2, c.T - 1
    n = len(s_idx)
    return _copy(c, stats=np.concatenate([osum.sum(axis=0), osq.sum(axis=0), [float(rows * n), float(n)]]))


def _act_forms_bug(c: Capture, which: str, xp) -> list:
    """The layer activations of ``c``'s policy evaluated wrongly on purpose: 'tanh_layer' tanh in the first hidden layer,
    'default_param' torch's default slope (0.01) or alpha (1.0) in place of the policy's, 'no_output' no activation after
    the output layer."""
    from es_pytorch_b200 import _lib
    from es_pytorch_b200.nn.nn import Activation
    acts = layer_forms(c, xp)
    if which == 'tanh_layer':
        acts[0] = xp.tanh
    elif which == 'default_param':
        default = {_lib.ES_ACT_LEAKY_RELU: 0.01, _lib.ES_ACT_ELU: 1.0}[int(c.activation.kind)]
        acts = [f64.form(Activation(c.activation.kind, default), xp)] * len(acts)
    else:
        acts[-1] = lambda z: z
    return acts


def _m_activation(c: Capture, which: str) -> Capture:
    """The fitness (and behaviour) of a rollout with ``_act_forms_bug(which)``, everything after it rescored: in the closed
    loop on the truth's sample, the pairs the fitness stage compares."""
    f = c.fit.copy()
    behv = None if c.behv is None else c.behv.copy()
    if c.closed:
        tr = closed_truth(c, growth=False, acts=_act_forms_bug(c, which, np))
        f[:, tr['pairs'], 0] = tr['fit']
        if behv is not None:
            behv[:, tr['pairs']] = tr['behv'].astype(F32)
    else:
        tf, tb, _, _ = fitness_truth(c, acts=_act_forms_bug(c, which, torch))
        f[:, :, 0] = tf
        if behv is not None:
            behv = tb.astype(F32)
    return _rescored(_copy(c, fit=f, behv=behv))


# name -> (what it models, mutation); each returns a mutated copy of a correct capture
MUTATIONS = {
    'shift_stream_indices': ("one stream's indices shifted by a pair", _m_shift_stream),
    'swap_stream_blocks': ("two streams' blocks swapped", _m_swap_streams),
    'plus_coin_on_minus': ('the + coin applied to the - evaluation', _m_coin_to_neg),
    'drop_save': ('one save dropped from the count', _m_drop_save),
    'sign_swap': ("one pair's signs swapped", _m_sign_swap),
    'novelty_column': ('novelty in the wrong column', _m_novelty_column),
    'novelty_off_by_one': ('novelty of the next evaluation', _m_novelty_off_by_one),
    'weights_next': ('weights paired with idx[k + 1]', _m_weights_next),
    'gsum_over_k': ('gsum divided by K instead of 2K', _m_gsum_over_k),
    'l2_sign': ("the l2 term's sign flipped", _m_l2_sign),
    'adam_t': ("Adam's t not advanced", _m_adam_t),
    'std_squared': ('normalisation by std^2', _m_std_squared),
    'stale_colsum': ('a stale column-sum cache from a previous obs stream', _m_stale_colsum),
    'episode0_noise': ("episode 0's noise reused for every episode", _m_ep0_noise),
    'episodes_not_divided': ('the episode sum not divided by E', _m_episodes_not_divided),
    'first_episode_behaviour': ('behaviour taken from the first episode', _m_first_episode_behaviour),
    'novelty_over_reward': ('novelty written to the reward column', _m_novelty_over_reward),
    'moo_w_swapped': ('the MultiObjective blend with w and 1 - w swapped', _m_moo_w_swapped),
    'archive_clipped_to_k': ('novelty averaged over k instead of min(k, A) archive entries', _m_archive_clipped),
    'closed_obstat_pre_step': ('closed-loop ObStat summed over obs_0 .. obs_{T-1}', lambda c: _closed_saved_sums(c, 'pre')),
    'closed_count_t_minus_1': ('closed-loop ObStat of T - 1 rows per saved evaluation', lambda c: _closed_saved_sums(c, 'short')),
    'closed_drop_saved': ('one saved evaluation dropped from the closed-loop ObStat', lambda c: _closed_saved_sums(c, drop=1)),
    'act_tanh_layer': ('tanh in place of the policy\'s activation in the first hidden layer',
                       lambda c: _m_activation(c, 'tanh_layer')),
    'act_default_param': ("torch's default slope (0.01) or alpha (1.0) in place of the policy's",
                          lambda c: _m_activation(c, 'default_param')),
    'act_no_output': ('no activation after the output layer', lambda c: _m_activation(c, 'no_output')),
}
NEEDS_ARCHIVE = ('novelty_column', 'novelty_off_by_one')
# what capture a mutation models a bug of, beyond a plain open-loop one: 'episodes' (E > 1 with action noise), 'nsr'
# (an archive; 'moo_w_swapped' needs w != 0.5, 'archive_clipped_to_k' fewer entries than k), 'closed' (the closed loop),
# 'activation' (a policy activation other than tanh, open or closed loop) and 'param' (leaky ReLU or ELU)
NEEDS = {'episode0_noise': 'episodes', 'episodes_not_divided': 'episodes', 'first_episode_behaviour': 'episodes',
         'novelty_over_reward': 'nsr', 'moo_w_swapped': 'nsr', 'archive_clipped_to_k': 'nsr',
         'closed_obstat_pre_step': 'closed', 'closed_count_t_minus_1': 'closed', 'closed_drop_saved': 'closed',
         'act_tanh_layer': 'activation', 'act_default_param': 'param', 'act_no_output': 'activation'}
ACT_MUTATIONS = ('act_tanh_layer', 'act_default_param', 'act_no_output')


def rejection(checks: Sequence[Check]):
    """(stages that failed, the largest margin among the failed checks) -- (None, 0) when everything passed."""
    bad = failed(checks)
    if not bad:
        return None, 0.0
    return sorted({c.stage for c in bad}, key=STAGES.index), max(c.margin for c in bad)
