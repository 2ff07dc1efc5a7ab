"""CPU oracle for the OpenAI-ES generation step of sash-a/es_pytorch.

TEST INFRASTRUCTURE ONLY.  Nothing under ``es_pytorch_b200/`` may import this
module; it is used by ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` as the *checker*
and as the timed CPU baseline, never as the product path.

It restates, function by function, the arithmetic of the reference's hot path
(SURVEY.md section 8a).  Every function cites the reference ``file:line`` it
follows (paths relative to the reference checkout).

Pinning status (SURVEY.md section 8c):
  * pinned by the reference's own known-answer tests (re-run in
    ``tests/test_oracle_golden.py``): ``scale_noise`` / ``batch_noise``
    (test/utils/utils_test.py:7-40), MOO rank blend (test/utils/rankers.py:6-27),
    ``_share_results`` row layout (test/es/es_runner_test.py:10-31), novelty
    (test/utils/novelty_test.py:27-33), obstat merge (test/utils/obstat_test.py:8-23),
    table content (test/es/noisetable_test.py:19-26);
  * pinned against the real reference modules that import in the build container
    (``src.utils.rankers``, ``src.nn.optimizers``): ``tests/golden/make_golden.py``
    ran them and committed the vectors -- ``ref_vectors.npz`` (CenteredRanker, MultiObjectiveRanker,
    SGD / Adam / SimpleES steps, legacy RandomState streams) and ``ref_rankers.npz`` (DoublePositiveCentered,
    SemiCentered, MaxNormalized, EliteRanker and their MultiObjective blends);
  * pinned against the REAL reference pipeline executed in the build container (``tests/golden/make_ref_pipeline.py``
    imports /root/reference's ``src.core.es`` / ``policy`` / ``noisetable`` / ``nn`` / ``gym_runner`` / ``training_result`` /
    ``obstat`` / ``optimizers`` with inert stand-ins for the absent mpi4py / gym / munch / mlflow and runs two generations;
    vectors in ``ref_pipeline.npz``): ``Policy.pheno``, ``FeedForward.forward``, ``run_model``, the RNG interleaving of
    ``test_params``, ``approx_grad``, ``Policy.update_obstat`` -- indices, obs statistics and rank weights reproduce
    bit-exactly, fitness to a float32 ulp (bit-exact with the same torch CPU threading), theta within 2e-6 (the real Adam computes a float64 step under numpy 2);
    The same file holds a real NSRA-style generation (``NSRResult`` + ``MultiObjectiveRanker(CenteredRanker(), 0.5)``) and
    a real ``EliteRanker(CenteredRanker(), 0.25)`` update (obj.py:50), two momentum-``SGD`` and ``SimpleES`` updates through
    the real ``approx_grad``, reproduced the same way;
    plus the real ``test_params`` on two thread-emulated MPI ranks (rank-major ``_share_results`` rows, per-rank RNG streams,
    summed steps, ``ObStat.mpi_inc``): what a process carrying two 'virtual ranks' must reproduce.

  * the CLOSED-LOOP synthetic env (``ClosedLoopEnvSpec``, stepped by ``run_model``) has no reference implementation
    (SURVEY.md section 8d names only the transition ``obs' = tanh(A obs + B a)``): for that variant, with its action noise
    and multi-episode evaluations, this module is the definition -- parity unpinned against the reference by construction;
    the noise-free single episode is frozen by ``tests/golden/closed_loop.npz``.
  * the binned head of FFBinned (``binned_action``, src/nn/nn.py:99-117) is pinned bit for bit against the package's
    ``FFBinned.forward`` by ``tests/test_binned_host.py``.

Float semantics are those of the reference's pinned stack (numpy 1.18 value-based
casting): every array op on float32 data stays float32 and python scalars are
rounded to float32 before the op.  Under numpy 2.x the real ``Adam`` would compute
its step in float64 (np.float64 scalar ``a``); the oracle pins the 1.18 behaviour
explicitly with casts so it is independent of the numpy that runs it.
"""
from __future__ import annotations

import heapq
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

F32 = np.float32


# ----------------------------------------------------------------------------
# noise table  (src/core/noisetable.py:27-64)
# ----------------------------------------------------------------------------
def make_noise(size: int, seed: int) -> np.ndarray:
    """Table content as the reference's own test asserts it
    (test/es/noisetable_test.py:26): legacy ``RandomState(seed).randn(size)`` cast
    to float32.  (noisetable.py:61-64 routes the seed through gym 0.17.1's
    ``np_random`` hash; gym is a third-party dep absent here, the two disagree, and
    parity harnesses therefore always pass the table in explicitly.)"""
    return np.random.RandomState(seed).randn(size).astype(F32)


def table_get(table: np.ndarray, i: int, size: int) -> np.ndarray:
    """noisetable.py:33-35 -- a *view*; asserts ``len > i + size``."""
    assert len(table) > i + size, 'trying to index outside the range of the noise table'
    return table[i:i + size]


def sample_idx(table_len: int, rs: np.random.RandomState, size: int) -> int:
    """noisetable.py:37-40 -- ``rs.randint(0, len - size)`` (legacy masked rejection)."""
    upper_bound = table_len - size
    if upper_bound <= 0:
        raise ValueError(f'Network (size:{size}) is too large for noise table (size:{table_len})')
    return int(rs.randint(0, upper_bound))


# A from-scratch MT19937 + legacy-randint restatement (numpy/random/_mt19937 and
# numpy/random/src/distributions: ``buffered_bounded_masked_uint32``; numpy 1.18.4,
# frozen by NEP 19).  Used to cross-check what the CUDA index-draw kernel has to
# reproduce word by word; numpy's RandomState itself is the primary oracle.
def mt_regen(mt: List[int]) -> List[int]:
    n, m = 624, 397
    mt = list(mt)
    for i in range(n):
        y = (mt[i] & 0x80000000) | (mt[(i + 1) % n] & 0x7FFFFFFF)
        mt[i] = mt[(i + m) % n] ^ (y >> 1) ^ (0x9908B0DF if (y & 1) else 0)
    return mt


def mt_temper(y: int) -> int:
    y ^= y >> 11
    y ^= (y << 7) & 0x9D2C5680
    y ^= (y << 15) & 0xEFC60000
    y ^= y >> 18
    return y & 0xFFFFFFFF


def mt_draw_indices(key: Sequence[int], pos: int, n: int, upper_bound: int, extra_words: int):
    """Replays ``n`` times: ``randint(0, upper_bound)`` then ``extra_words`` raw
    32-bit outputs (e.g. 4 = the two ``rs.random()`` save_obs coins that
    simple_example.py:38 draws per antithetic pair, es.py:68-72).
    Returns (indices, extras[n][extra_words], new_key, new_pos)."""
    mt = [int(x) for x in key]
    rng = upper_bound - 1
    mask = rng
    for s in (1, 2, 4, 8, 16):
        mask |= mask >> s
    assert 0 < rng < 0xFFFFFFFF

    def next32():
        nonlocal mt, pos
        if pos == 624:
            mt = mt_regen(mt)
            pos = 0
        w = mt_temper(mt[pos])
        pos += 1
        return w

    idx, extras = [], []
    for _ in range(n):
        while True:
            v = next32() & mask
            if v <= rng:
                break
        idx.append(v)
        extras.append([next32() for _ in range(extra_words)])
    return idx, extras, mt, pos


def words_to_double(a: int, b: int) -> float:
    """legacy ``random_sample``: 53-bit double from two 32-bit words."""
    return ((a >> 5) * 67108864.0 + (b >> 6)) / 9007199254740992.0


# ----------------------------------------------------------------------------
# policy: flat params <-> layers, perturbation (src/core/policy.py:33-35,49-67)
# ----------------------------------------------------------------------------
def layer_dims(obs_dim: int, hidden: Sequence[int], act_dim: int) -> List[Tuple[int, int]]:
    """nn.py:32-36 -- Linear(in,out) for consecutive sizes, activation after each."""
    sizes = [int(obs_dim)] + [int(h) for h in hidden] + [int(act_dim)]
    return list(zip(sizes[:-1], sizes[1:]))


def n_params(dims: Sequence[Tuple[int, int]]) -> int:
    return sum(i * o + o for i, o in dims)


def unflatten(params: np.ndarray, dims: Sequence[Tuple[int, int]]):
    """policy.py:49-59 -- state_dict order: weight[out,in] row-major, then bias[out]."""
    out, off = [], 0
    for i, o in dims:
        w = params[off:off + i * o].reshape(o, i)
        off += i * o
        b = params[off:off + o]
        off += o
        out.append((w, b))
    assert off == len(params)
    return out


def pheno_params(flat: np.ndarray, std: float, noise: Optional[np.ndarray]) -> np.ndarray:
    """policy.py:61-64 -- ``flat + std * noise``: two separately rounded float32 ops
    (no fused multiply-add) when noise is float32; the noiseless call passes float64
    zeros (es.py:48) which leaves the float32 values unchanged."""
    flat = np.asarray(flat, dtype=F32)
    if noise is None:
        return flat.copy()
    noise = np.asarray(noise)
    if noise.dtype == F32:
        return (flat + (F32(std) * noise).astype(F32)).astype(F32)
    return (flat.astype(np.float64) + float(std) * noise.astype(np.float64)).astype(F32)


# ----------------------------------------------------------------------------
# forward (src/nn/nn.py:42-50)
# ----------------------------------------------------------------------------
def normalise_obs(ob: np.ndarray, obmean: np.ndarray, obstd: np.ndarray, ob_clip: float) -> np.ndarray:
    """nn.py:45 -- float32 tensor minus float64 ndarray promotes to float64 in torch;
    clamp; then ``.float()``."""
    x = (np.asarray(ob, dtype=F32).astype(np.float64) - np.asarray(obmean, np.float64)) / np.asarray(obstd, np.float64)
    return np.clip(x, -float(ob_clip), float(ob_clip)).astype(F32)


def mlp_forward(layers, x: np.ndarray) -> np.ndarray:
    """nn.py:46 -- Sequential(Linear, Tanh, ...), activation after *every* layer
    including the output.  ``x`` is [obs] or [B, obs] float32."""
    import torch
    h = torch.from_numpy(np.ascontiguousarray(x, dtype=F32))
    with torch.no_grad():
        for w, b in layers:
            h = torch.tanh(torch.nn.functional.linear(h, torch.from_numpy(np.ascontiguousarray(w)),
                                                      torch.from_numpy(np.ascontiguousarray(b))))
    return h.numpy()


# ----------------------------------------------------------------------------
# synthetic open-loop vector env + rollout (src/gym/gym_runner.py:33-67)
# ----------------------------------------------------------------------------
@dataclass
class SyntheticEnvSpec:
    """The synthetic env of SURVEY.md section 8d: observations are an open-loop
    stream shared by all policies, reward r_t = <a_t, c_t>, the 'robot position'
    integrates the first three action components.  ``obs_stream`` has T+1 rows: row
    t is what the policy sees at step t, row t+1 is what ``env.step`` returns."""
    obs_dim: int
    act_dim: int
    T: int
    obs_seed: int = 11
    rew_seed: int = 13
    pos_scale: float = 0.05
    obs_stream: np.ndarray = field(init=False, repr=False)
    rew_vec: np.ndarray = field(init=False, repr=False)

    def __post_init__(self):
        self.obs_stream = np.random.RandomState(self.obs_seed).randn(self.T + 1, self.obs_dim).astype(F32)
        self.rew_vec = np.random.RandomState(self.rew_seed).randn(self.T, self.act_dim).astype(F32)


@dataclass
class ClosedLoopEnvSpec(SyntheticEnvSpec):
    """The closed-loop variant SURVEY.md section 8d names as optional (labelled separately everywhere):
    ``obs_{t+1} = tanh(A obs_t + B a_t)`` with a banded, wrap-around A (``band`` diagonals centred on the main one) and a
    dense B; obs_0 = row 0 of the open-loop stream; reward and position as in the open-loop env.  All float32; the
    pre-activation is accumulated in index order (A's diagonals, then B's columns), products and sums rounded separately."""
    band: int = 8
    a_seed: int = 17
    b_seed: int = 19
    a_gain: float = 0.5
    b_gain: float = 0.5
    closed_loop: bool = field(init=False, default=True)
    env_a: np.ndarray = field(init=False, repr=False)        # [obs][band]
    env_b: np.ndarray = field(init=False, repr=False)        # [obs][act]

    def __post_init__(self):
        super().__post_init__()
        self.env_a = (np.random.RandomState(self.a_seed).randn(self.obs_dim, self.band) *
                      (self.a_gain / np.sqrt(self.band))).astype(F32)
        self.env_b = (np.random.RandomState(self.b_seed).randn(self.obs_dim, self.act_dim) *
                      (self.b_gain / np.sqrt(self.act_dim))).astype(F32)

    def step_obs(self, ob: np.ndarray, a: np.ndarray) -> np.ndarray:
        n, half = self.obs_dim, self.band // 2
        ob, a = np.asarray(ob, dtype=F32), np.asarray(a, dtype=F32)
        acc = np.zeros(n, dtype=F32)
        for d in range(self.band):
            acc = (acc + (self.env_a[:, d] * np.roll(ob, half - d)).astype(F32)).astype(F32)     # ob[(i + d - half) % n]
        for j in range(self.act_dim):
            acc = (acc + (self.env_b[:, j] * a[j]).astype(F32)).astype(F32)
        return np.tanh(acc).astype(F32)


def binned_action(out: np.ndarray, bins: int, low: np.ndarray, high: np.ndarray) -> np.ndarray:
    """FFBinned's head (nn.py:99-117): [..., adim * bins] network outputs -> [..., adim] float32 actions.  The first maximal
    bin of each dimension (numpy's argmax, like torch's, returns the first), then, with float32 ``low`` / ``high`` (the env's
    Box), ``((c * idx) * range) + low`` with ``c = float32(1 / (bins - 1))``, every operation rounded to float32 as torch
    evaluates it."""
    out = np.asarray(out, dtype=F32)
    low = np.asarray(low, dtype=F32)
    rng = (np.asarray(high, dtype=F32) - low).astype(F32)
    idx = out.reshape(out.shape[:-1] + (low.shape[0], int(bins))).argmax(-1)
    c = F32(1.0 / (bins - 1.0))
    return (((c * idx.astype(F32)).astype(F32) * rng).astype(F32) + low).astype(F32)


def run_model(env: SyntheticEnvSpec, layers, obmean, obstd, ob_clip: float, max_steps: int,
              batched: bool = False, ac_std: float = 0.0, rs: Optional[np.random.RandomState] = None,
              episodes: int = 1, binned: Optional[Tuple[int, np.ndarray, np.ndarray]] = None):
    """gym_runner.py:33-67 on the synthetic envs, inside obj.py:54-63's ``eps_per_policy`` loop.  Returns (rews list,
    behv list (3 per step, padded), obs ndarray [steps, obs_dim] of post-step observations, step = last loop index).

    Every step: forward the normalised observation (nn.py:42-50), add the action noise, reward ``<a_t, c_t>`` as a float32
    dot in index order, integrate the position from the first three action components, and on the closed loop
    (``env.closed_loop``) step the env with the action.  The open loop's observations do not depend on the actions, so
    its forwards run before the steps: ``batched=True`` evaluates them in one matrix product (same arithmetic up to BLAS
    summation order) so large parity cases finish in seconds; otherwise one forward per step, the literal restatement.

    ``ac_std != 0`` with a stream ``rs``: FeedForward.forward adds ``rs.randn(*a.shape) * ac_std`` to the action at every
    step (nn.py:47-48; legacy polar-method gaussians from the SAME RandomState that draws the noise indices and the
    save_obs coins).  ``a += ndarray`` on a float32 tensor yields the float64 sum (numpy's reflected add wraps the
    result back into a tensor), which the env casts to float32 (``np.asarray(action, dtype=float32)``).

    ``binned=(bins, low, high)``: FFBinned's head (``binned_action``) in place of the tanh output.  FFBinned.forward ignores
    ``rs``, so a binned policy draws no noise.

    ``episodes=E``: ``max(1, E)`` episodes from a fresh env, each drawing its own noise; as obj.py:57-60, the rewards are
    summed per step into a float64 array of ``max_steps`` zeros in episode order and divided by the count.  Behaviour,
    observations and step are the last episode's.  One episode returns its own reward list, unpadded."""
    closed = getattr(env, 'closed_loop', False)
    n = min(int(max_steps), env.T)

    def forward(x):
        out = mlp_forward(layers, x)
        return out if binned is None else binned_action(out, *binned)

    if not closed:
        xs = normalise_obs(env.obs_stream[:n], obmean, obstd, ob_clip)
        acts = forward(xs) if batched else np.stack([forward(xs[t]) for t in range(n)])
    noisy = binned is None and ac_std != 0 and rs is not None
    ps = F32(env.pos_scale)
    n_eps = max(1, int(episodes))
    total = np.zeros(int(max_steps))
    for _ in range(n_eps):
        rews, behv, obs = [], [], []
        pos = np.zeros(3, dtype=F32)
        ob = env.obs_stream[0].copy()
        for t in range(n):
            a = (forward(normalise_obs(ob, obmean, obstd, ob_clip)) if closed else acts[t]).astype(F32)
            if noisy:
                a = (a.astype(np.float64) + rs.randn(env.act_dim) * ac_std).astype(F32)
            acc = F32(0.0)
            for j in range(env.act_dim):           # float32 dot, index order
                acc = F32(acc + F32(a[j] * env.rew_vec[t, j]))
            rews.append(float(acc))
            for j in range(3):
                pos[j] = F32(pos[j] + F32(ps * a[j % env.act_dim]))
            behv.extend([float(pos[0]), float(pos[1]), float(pos[2])])
            if closed:
                ob = env.step_obs(ob, a)
                obs.append(ob)
        total[:n] += np.array(rews)
    behv += behv[-3:] * (max_steps - int(len(behv) / 3))
    obs = np.stack(obs) if closed else env.obs_stream[1:n + 1].copy()
    if n_eps > 1:
        rews = (total / n_eps).tolist()
    return rews, behv, obs, n - 1                # gym_runner.py:50,67 returns the loop index


def _rollout_kw(episodes: int, binned) -> dict:
    """The ``episodes`` / ``binned`` keywords the generation functions pass to ``run_model``, left out at their defaults.
    A single tanh episode is then ``run_model``'s original nine-argument call, so a caller that substitutes its own
    rollout with that signature for ``run_model`` keeps working."""
    kw = {} if episodes == 1 else dict(episodes=episodes)
    if binned is not None:
        kw['binned'] = binned
    return kw


def reward_result(rews: List[float]) -> List[float]:
    """training_result.py:28,62-64 -- python ``sum`` (sequential float64)."""
    return [sum(rews)]


def novelty(behaviour: np.ndarray, archive: np.ndarray, k: int) -> float:
    """novelty.py:16-18 -- mean of the k smallest euclidean distances (k clipped to
    the archive size by ``heapq.nsmallest``)."""
    b = np.asarray(behaviour, dtype=np.float64)
    a = np.asarray(archive, dtype=np.float64)
    d = np.sqrt(((a - b[None, :]) ** 2).sum(axis=1))
    return float(np.mean(heapq.nsmallest(k, d)))


def nsr_result(rews: List[float], behv: List[float], archive: np.ndarray, k: int) -> List[float]:
    """training_result.py:29,82-97 -- [sum(rewards), novelty(positions[-3:-1])]."""
    return [sum(rews), novelty(np.array(behv[-3:-1]), archive, k)]


def ob_sum_sq_cnt(obs: np.ndarray):
    """training_result.py:17-21."""
    cnt = len(obs) if np.any(obs) else 0
    return obs.sum(axis=0), np.square(obs).sum(axis=0), cnt


# ----------------------------------------------------------------------------
# obs statistics (src/nn/obstat.py:13-37)
# ----------------------------------------------------------------------------
class ObStatOracle:
    def __init__(self, shape, eps):
        self.sum = np.zeros(shape, dtype=np.float64)
        self.sumsq = np.full(shape, eps, dtype=np.float64)
        self.count = eps

    def inc(self, s, ssq, c):
        self.sum += np.asarray(s).astype(np.float64)
        self.sumsq += np.asarray(ssq).astype(np.float64)
        self.count += c

    def merge(self, other: 'ObStatOracle'):
        self.inc(other.sum, other.sumsq, other.count)

    @property
    def mean(self):
        return self.sum / self.count

    @property
    def std(self):
        return np.sqrt(np.maximum(self.sumsq / self.count - np.square(self.mean), 1e-2))


# ----------------------------------------------------------------------------
# ES generation: sampling loop + result sharing (src/core/es.py:54-95)
# ----------------------------------------------------------------------------
def share_results(per_rank_rows: List[np.ndarray]) -> np.ndarray:
    """es.py:84-95 -- every rank tiles its rows ``size`` times and Alltoall's them,
    i.e. an allgather: the result is the rank-major concatenation of the per-rank
    ``[fits_pos..., fits_neg..., idx]`` rows, float64."""
    return np.concatenate([np.asarray(r, dtype=np.float64) for r in per_rank_rows], axis=0)


def es_test_params(table: np.ndarray, flat: np.ndarray, std: float, dims, env: SyntheticEnvSpec,
                rank_seeds: Sequence[int], n_per_rank: int, obmean, obstd, ob_clip: float,
                max_steps: int, coins_per_eval: int = 0, save_obs_chance: float = 0.0,
                archive: Optional[np.ndarray] = None, nov_k: int = 10, batched: bool = True,
                rank_states: Optional[List[np.random.RandomState]] = None, ac_std: float = 0.0,
                episodes: int = 1, binned=None):
    """es.py:54-81 replayed for R virtual MPI ranks (one legacy RandomState per rank,
    utils.py:63-65).  Per pair: ``nt.sample(rs)`` (one ``randint``), evaluate +noise,
    evaluate -noise (es.py:68-72); each evaluation's fit_fn draws ``coins_per_eval``
    ``rs.random()`` values first (1 in simple_example.py:38 / obj.py:54, 0 for the
    index-only variant), then runs ``run_model`` with ``episodes`` and ``binned``.
    Returns (pos[K,n_obj], neg[K,n_obj], inds[K], steps, obstat) with K = R*n_per_rank
    in rank-major order, all float64 like es.py:89."""
    P = len(flat)
    n_obj = 1 if archive is None else 2
    gen_obstat = ObStatOracle((env.obs_dim,), 0)
    rows_per_rank, steps_total = [], 0
    for r, seed in enumerate(rank_seeds):
        rs = rank_states[r] if rank_states is not None else np.random.RandomState(seed)
        rows = []
        for _ in range(n_per_rank):
            idx = sample_idx(len(table), rs, P)
            noise = table_get(table, idx, P)
            res = []
            for sign in (1.0, -1.0):
                save_obs = False
                for _c in range(coins_per_eval):
                    save_obs = rs.random() < save_obs_chance
                layers = unflatten(pheno_params(flat, std, noise if sign > 0 else -noise), dims)
                rews, behv, obs, step = run_model(env, layers, obmean, obstd, ob_clip, max_steps, batched, ac_std, rs,
                                                  **_rollout_kw(episodes, binned))
                res.append(reward_result(rews) if archive is None else nsr_result(rews, behv[-3:], archive, nov_k))
                steps_total += step
                o = obs if save_obs else np.array([np.zeros((env.obs_dim,))])
                gen_obstat.inc(*ob_sum_sq_cnt(o))
            rows.append(res[0] + res[1] + [idx])
        rows_per_rank.append(np.array(rows, dtype=np.float64).reshape(n_per_rank, 2 * n_obj + 1))
    results = share_results(rows_per_rank)
    return results[:, 0:n_obj], results[:, n_obj:2 * n_obj], results[:, -1], steps_total, gen_obstat


# ----------------------------------------------------------------------------
# rank transforms (src/utils/rankers.py:9-58,106-120)
# ----------------------------------------------------------------------------
def rank(x: np.ndarray) -> np.ndarray:
    """rankers.py:9-17.  Ties: the reference's ``argsort()`` is an unstable sort so
    tie order is unpinned; the oracle (and the CUDA kernel) define it as
    stable-by-position, which is what ``kind='stable'`` gives."""
    assert x.ndim == 1
    ranks = np.empty(len(x), dtype=np.int64)
    ranks[np.argsort(x, kind='stable')] = np.arange(len(x))
    return ranks


def centered_rank(x: np.ndarray) -> np.ndarray:
    """rankers.py:53-58 -- float32(rank) / (size-1) - 0.5, both ops in float32."""
    y = rank(x.ravel()).reshape(x.shape).astype(F32)
    y = (y / F32(x.size - 1)).astype(F32)
    y = (y - F32(0.5)).astype(F32)
    return np.squeeze(y)


def centered_ranker(fits_pos: np.ndarray, fits_neg: np.ndarray):
    """Ranker.rank with CenteredRanker (rankers.py:30,37-50): concat pos,neg ->
    rank -> pos part minus neg part.  Returns (weights float32[K], n_fits_ranked)."""
    fits = np.concatenate((fits_pos, fits_neg))
    y = centered_rank(fits)
    k = len(fits_pos)
    return (y[:k] - y[k:]).astype(F32), int(y.size)


def moo_ranker(fits_pos: np.ndarray, fits_neg: np.ndarray, w: float):
    """MultiObjectiveRanker over CenteredRanker (rankers.py:106-120): exactly two
    objective columns, each ranked independently, blended ``r0*w + r1*(1-w)`` with the
    python floats rounded to float32 by the array op."""
    fits = np.concatenate((fits_pos, fits_neg))
    assert fits.shape[1] == 2
    r0 = centered_rank(fits[:, 0])
    r1 = centered_rank(fits[:, 1])
    y = ((r0 * F32(w)).astype(F32) + (r1 * F32(1 - w)).astype(F32)).astype(F32)
    k = len(fits_pos)
    return (y[:k] - y[k:]).astype(F32), int(y.size)


def double_positive_rank(x: np.ndarray) -> np.ndarray:
    """DoublePositiveCenteredRanker._rank, rankers.py:61-65: centered ranks, positive half times two (float32)."""
    y = np.array(centered_rank(x), dtype=F32, copy=True)
    y[y > 0] = (y[y > 0] * F32(2)).astype(F32)
    return y


def max_normalized(x: np.ndarray) -> np.ndarray:
    """MaxNormalizedRanker._rank, rankers.py:68-75 (float64; the shift ADDS a non-positive minimum, as written)."""
    x = np.asarray(x, dtype=np.float64)
    mn = np.min(x)
    y = x + (-mn if mn > 0 else mn)
    y = y / np.max(y)
    y = 2 * y - 1
    return np.squeeze(y)


def semi_centered_rank(x: np.ndarray) -> np.ndarray:
    """SemiCenteredRanker._rank, rankers.py:78-83: every python-float operand is rounded to float32 by the array
    operation (numpy 1.18 value-based casting and numpy 2 weak scalars agree); no squeeze."""
    y = rank(x.ravel()).reshape(x.shape).astype(F32)
    s = x.size
    t = (y + F32(0.29 * s)).astype(F32)
    u = (F32(1 / s) * np.square(t).astype(F32)).astype(F32)
    return ((u / F32(s)).astype(F32) - F32(0.5)).astype(F32)


SHAPINGS = {'centered': centered_rank, 'double_positive': double_positive_rank, 'max_normalized': max_normalized,
            'semi_centered': semi_centered_rank}


def shaped_ranker(fits_pos: np.ndarray, fits_neg: np.ndarray, shaping: str, w: Optional[float] = None):
    """Ranker.rank (rankers.py:37-50) for any plain shaping; ``w`` not None = MultiObjectiveRanker(shaping, w)
    (rankers.py:106-120).  Returns (ranked_fits, n_fits_ranked) with the reference's dtype."""
    fn_ = SHAPINGS[shaping]
    fits = np.concatenate((fits_pos, fits_neg))
    if w is None:
        y = fn_(fits)
    else:
        assert fits.shape[1] == 2
        r0, r1 = fn_(fits[:, 0]), fn_(fits[:, 1])
        y = r0 * w + r1 * (1 - w)            # python floats: the arrays keep their dtype (float32 / float64)
        y = y.astype(r0.dtype)
    k = len(fits_pos)
    return y[:k] - y[k:], int(y.size)


def elite_ranker(fits_pos: np.ndarray, fits_neg: np.ndarray, noise_inds: np.ndarray, shaping: str,
                 elite_percent: float):
    """EliteRanker(shaping, elite_percent).rank, rankers.py:86-103: the n_elite largest shaped values, unsubtracted,
    with ``noise_inds[fit_index % K]``.  np.argpartition's order is unspecified; returned in ascending (stable) order
    of the shaped values (note: max_normalized DEcreases with the fitness when max + min < 0, rankers.py:71-72).  Returns (ranked_fits[n_elite], noise_inds[n_elite], fit_index[n_elite], n_elite)."""
    fits = np.concatenate((fits_pos, fits_neg))
    ranked = np.asarray(SHAPINGS[shaping](fits)).ravel()
    n_elite = max(1, int(ranked.size * elite_percent))
    order = np.argsort(ranked, kind='stable')                      # fit indices by ascending shaped value
    elite = order[-n_elite:]
    return ranked[elite], np.asarray(noise_inds)[elite % len(noise_inds)], elite, n_elite


# ----------------------------------------------------------------------------
# gradient reconstruction (src/utils/utils.py:14-39) and update (es.py:98-101)
# ----------------------------------------------------------------------------
def batch_noise(inds: np.ndarray, table: np.ndarray, policy_len: int, batch_size: int):
    """utils.py:14-26 -- dense [B,P] copies of the slices, B <= batch_size."""
    assert inds.ndim == 1
    batch = []
    for idx in inds:
        batch.append(table_get(table, int(idx), policy_len))
        if len(batch) == batch_size:
            yield np.array(batch)
            batch = []
    if batch:
        yield np.array(batch)


def scale_noise(fits: np.ndarray, noise_inds: np.ndarray, table: np.ndarray, policy_len: int,
                batch_size: int) -> np.ndarray:
    """utils.py:29-39 -- sum over batches of ``dot(w[B], N[B,P])``."""
    assert len(fits) == len(noise_inds)
    total = 0
    for i, nb in zip(range(0, len(fits), batch_size), batch_noise(noise_inds, table, policy_len, batch_size)):
        total = total + np.dot(fits[i:min(i + batch_size, len(fits))], nb)
    return total


def scale_noise_f64(fits, noise_inds, table, policy_len) -> np.ndarray:
    """Same sum in float64 -- the 'true' value the 1e-5 rel tolerance is judged by."""
    total = np.zeros(policy_len, dtype=np.float64)
    for w, idx in zip(fits, noise_inds):
        total += float(w) * table[int(idx):int(idx) + policy_len].astype(np.float64)
    return total


class AdamOracle:
    """optimizers.py:13-21,47-61 with numpy-1.18 casting pinned: m, v, step float32;
    python-float scalars (beta, 1-beta, a, epsilon) rounded to float32 by each op."""

    def __init__(self, dim, lr, beta1=0.9, beta2=0.999, epsilon=1e-08):
        self.lr, self.dim, self.t = lr, dim, 0
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon
        self.m = np.zeros(dim, dtype=F32)
        self.v = np.zeros(dim, dtype=F32)

    def step(self, g: np.ndarray) -> np.ndarray:
        g = np.asarray(g, dtype=F32)
        self.t += 1
        a = self.lr * np.sqrt(1 - self.beta2 ** self.t) / (1 - self.beta1 ** self.t)   # python/np float64 scalar
        self.m = (F32(self.beta1) * self.m + F32(1 - self.beta1) * g).astype(F32)
        self.v = (F32(self.beta2) * self.v + F32(1 - self.beta2) * (g * g)).astype(F32)
        return ((F32(-a) * self.m) / (np.sqrt(self.v) + F32(self.epsilon))).astype(F32)


class SGDOracle:
    """optimizers.py:36-44."""

    def __init__(self, dim, lr, momentum=0.9):
        self.lr, self.dim, self.t, self.momentum = lr, dim, 0, momentum
        self.v = np.zeros(dim, dtype=F32)

    def step(self, g):
        g = np.asarray(g, dtype=F32)
        self.t += 1
        self.v = (F32(self.momentum) * self.v + F32(1. - self.momentum) * g).astype(F32)
        return (F32(-self.lr) * self.v).astype(F32)


class SimpleESOracle:
    """optimizers.py:28-33."""

    def __init__(self, dim, lr):
        self.lr, self.dim, self.t = lr, dim, 0

    def step(self, g):
        self.t += 1
        return (F32(self.lr) * np.asarray(g, dtype=F32)).astype(F32)


def approx_grad(flat: np.ndarray, optim, ranked_fits: np.ndarray, noise_inds: np.ndarray, n_fits_ranked: int,
                table: np.ndarray, batch_size: int, l2coeff: float) -> np.ndarray:
    """es.py:98-101 + policy.py:73-74: grad = scale_noise / n_fits_ranked (no 1/sigma);
    flat += optim.step(l2coeff * flat - grad).  Mutates and returns ``flat``."""
    total = np.asarray(scale_noise(ranked_fits, noise_inds, table, len(flat), batch_size), dtype=F32)
    grad = (total / F32(n_fits_ranked)).astype(F32)
    g = ((F32(l2coeff) * flat).astype(F32) - grad).astype(F32)
    flat += optim.step(g)
    return flat


def generation(table, flat, optim, std, dims, env, rank_seeds, n_per_rank, obmean, obstd, ob_clip, max_steps,
               batch_size, l2coeff, moo_w: Optional[float] = None, archive=None, nov_k=10,
               coins_per_eval=0, rank_states=None, batched=True, shaping: str = 'centered',
               elite_percent: Optional[float] = None, save_obs_chance: float = 0.0, ac_std: float = 0.0,
               episodes: int = 1, binned=None):
    """One whole generation (es.py:38-47 without the reporter / noiseless eval).  ``shaping`` / ``elite_percent`` select
    the other rankers of rankers.py:61-103 (obj.py:48-50 picks EliteRanker(CenteredRanker(), elite))."""
    pos, neg, inds, steps, obstat = es_test_params(table, flat, std, dims, env, rank_seeds, n_per_rank, obmean, obstd,
                                                ob_clip, max_steps, coins_per_eval=coins_per_eval, archive=archive,
                                                nov_k=nov_k, batched=batched, rank_states=rank_states,
                                                save_obs_chance=save_obs_chance, ac_std=ac_std, episodes=episodes,
                                                binned=binned)
    grad_inds = inds
    if elite_percent is not None:
        w, grad_inds, _, n_ranked = elite_ranker(pos, neg, inds, shaping, elite_percent)
    elif shaping != 'centered':
        w, n_ranked = shaped_ranker(pos, neg, shaping, None if archive is None else moo_w)
        w = np.asarray(w).reshape(-1)
    elif archive is None:
        w, n_ranked = centered_ranker(pos, neg)
    else:
        w, n_ranked = moo_ranker(pos, neg, moo_w)
    approx_grad(flat, optim, w, grad_inds, n_ranked, table, batch_size, l2coeff)
    return dict(pos=pos, neg=neg, inds=inds, steps=steps, weights=w, n_ranked=n_ranked, obstat=obstat)


def es_step(table, flat, optim, std, dims, env, rank_states, n_per_rank, obmean, obstd, ob_clip, max_steps, batch_size,
            l2coeff, coins_per_eval=1, save_obs_chance=0.0, batched=True, episodes=1, binned=None, **kw):
    """``es.step`` (es.py:38-51): the generation, then the noiseless evaluation ``fit_fn(policy.pheno(zeros), False)`` of the
    UPDATED parameters that every rank runs for itself.  The scripts' fit_fn draws its save_obs coin(s) in every call
    (simple_example.py:38, obj.py:54), so each rank's stream advances by ``coins_per_eval`` doubles here too, and it runs
    its ``episodes`` whether or not it adds noise (obj.py:57).  Returns the generation's dict plus ``noiseless`` (the result
    list of rank 0)."""
    out = generation(table, flat, optim, std, dims, env, [None] * len(rank_states), n_per_rank, obmean, obstd, ob_clip,
                     max_steps, batch_size, l2coeff, coins_per_eval=coins_per_eval, rank_states=rank_states, batched=batched,
                     save_obs_chance=save_obs_chance, episodes=episodes, binned=binned, **kw)
    noiseless = None
    for rs in rank_states:
        for _c in range(coins_per_eval):
            rs.random()
        layers = unflatten(pheno_params(flat, std, None), dims)
        rews, behv, obs, step = run_model(env, layers, obmean, obstd, ob_clip, max_steps, batched,
                                          **_rollout_kw(episodes, binned))
        res = reward_result(rews) if kw.get('archive') is None else nsr_result(rews, behv[-3:], kw['archive'], kw.get('nov_k', 10))
        noiseless = res if noiseless is None else noiseless
    out['noiseless'] = noiseless
    return out
