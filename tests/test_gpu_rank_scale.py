"""es_rank_transform against the oracle's stable ranks (orc.rank, shaped_ranker, elite_ranker) at the benchmarked population sizes
and on fitness distributions that defeat rank.cu's linear value buckets: one outlier (every other value in one bucket), all equal,
+-1e308 (the span overflows), integers with thousands of ties, subnormals with +-0 (8192 / span overflows), values on exact bucket
edges, and infinities / NaN.  Every comparison is bit-exact: ranks, weights, weights64 and the elite lists (NaN compared as NaN).
Every case is also split into 2, 3 and 8 uneven shards; each shard must return its slice of the whole.

max_normalized decreases with the fitness when max + min < 0 (the integers in -9..0, all equal and negative): its elite then
orders equal fitnesses by ascending index, as a stable sort of the shaped values does.  With a NaN or -inf fitness every
max_normalized value is NaN (numpy's min and max propagate them) and the elite is the last elements by index.  Out of scope: a
+inf fitness among finite ones maps every finite fitness to -1, and the elite among those equal values follows the fitness, not the
index (distinct fitnesses with equal shaped values); only its values are compared there.  One outlier at 1e300 does the same:
every other fitness maps to exactly -1.
"""
import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu

SHAPINGS = ('centered', 'double_positive', 'semi_centered', 'max_normalized')
DISTS = ('gaussian', 'outlier', 'equal', 'equal_neg', 'huge', 'int_neg', 'int_pos', 'subnormal', 'bucket_edges', 'nan_inf',
         'neg_inf', 'pos_inf')
SIZES = (4800, 10000, 40000)
W_MOO = 0.37


def fitnesses(dist: str, K: int, n_obj: int, seed: int):
    rs = np.random.RandomState(seed)
    n = (2 * K, n_obj)
    if dist == 'gaussian':
        x = rs.randn(*n) * 10 + 1
    elif dist == 'outlier':
        x = rs.randn(*n)
        x[rs.randint(2 * K)] = 1e300
    elif dist == 'equal':
        x = np.full(n, 3.5)
    elif dist == 'equal_neg':
        x = np.full(n, -2.5)
    elif dist == 'huge':
        x = np.where(rs.rand(*n) < 0.5, -1e308, 1e308)
    elif dist == 'int_neg':
        x = rs.randint(-9, 1, n).astype(np.float64)
    elif dist == 'int_pos':
        x = rs.randint(0, 10, n).astype(np.float64)
    elif dist == 'subnormal':
        x = rs.randint(-40, 41, n) * 5e-324
        x[rs.rand(*n) < 0.2] = 0.0
        x[rs.rand(*n) < 0.2] = -0.0
        x[rs.rand(*n) < 0.05] = 2.5e-310
    elif dist == 'bucket_edges':
        mn, mx = -3.0, 5.0
        span = mx - mn
        x = mn + rs.randint(0, 8193, n) * span / 8192
        x[0], x[1] = mn, mx
    else:
        x = rs.randn(*n)
        m = rs.rand(*n)
        if dist == 'nan_inf':
            x[m < 0.01] = np.nan
            x[(m >= 0.01) & (m < 0.02)] = np.inf
            x[(m >= 0.02) & (m < 0.03)] = -np.inf
        elif dist == 'neg_inf':
            x[m < 0.02] = -np.inf
        else:
            x[m < 0.02] = np.inf
    return x[:K].copy(), x[K:].copy()


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == 'f')


def _kind(name):
    from es_pytorch_b200 import _lib
    return getattr(_lib, 'ES_RANK_' + name.upper())


def _shards(K, n, seed):
    cuts = np.sort(np.random.RandomState(seed).choice(np.arange(1, K), n - 1, replace=False))
    b = [0, *cuts.tolist(), K]
    return [(b[i], b[i + 1] - b[i]) for i in range(n)]


def _oracle_weights(pos, neg, name, n_obj):
    with np.errstate(all='ignore'):
        ref, _ = orc.shaped_ranker(pos, neg, name, None if n_obj == 1 else W_MOO)
    return np.asarray(ref, dtype=np.float64).reshape(-1)


@pytest.mark.parametrize('n_obj', [1, 2])
@pytest.mark.parametrize('dist', DISTS)
@pytest.mark.parametrize('K', SIZES)
def test_ranks_and_weights_exact_with_shards(eng, K, dist, n_obj):
    pos, neg = fitnesses(dist, K, n_obj, seed=K + 31 * DISTS.index(dist) + n_obj)
    full = np.concatenate((pos, neg))
    fp, fn = eng.to_device(pos), eng.to_device(neg)
    w0, w1 = (1.0, 0.0) if n_obj == 1 else (W_MOO, 1 - W_MOO)
    ref_ranks = np.stack([orc.rank(full[:, c]) for c in range(n_obj)])
    for name in SHAPINGS:
        ref = _oracle_weights(pos, neg, name, n_obj)
        out = eng.rank_transform(fp, fn, _kind(name), w0, w1, want64=True, want_ranks=True)
        got64 = out['weights64'].cpu().numpy()
        ranks = out['ranks'].cpu().numpy().reshape(n_obj, 2 * K)
        assert np.array_equal(ranks, ref_ranks), (name, dist)
        assert _same(got64, ref), (name, dist, np.flatnonzero(~((got64 == ref) | (np.isnan(got64) & np.isnan(ref))))[:5])
        assert _same(out['weights'].cpu().numpy(), ref.astype(np.float32)), (name, dist)
        for N in (2, 3, 8):
            for b, cnt in _shards(K, N, K + N):
                part = eng.rank_transform(fp, fn, _kind(name), w0, w1, k_begin=b, k_count=cnt, want64=True, want_ranks=True)
                assert _same(part['weights64'].cpu().numpy(), got64[b:b + cnt]), (name, N, b)
                pr = part['ranks'].cpu().numpy()
                assert np.array_equal(pr, ranks.reshape(n_obj, 2, K)[:, :, b:b + cnt]), (name, N, b)


def _check_elite(out, vals, sel, fit, K, name, fit_order_defined):
    assert _same(out['elite_vals'].cpu().numpy(), np.asarray(vals, dtype=np.float64)), name
    if fit_order_defined:
        assert np.array_equal(out['elite_fit'].cpu().numpy(), fit), name
        assert np.array_equal(out['elite_idx'].cpu().numpy(), sel), name


@pytest.mark.parametrize('pct', [0.01, 0.1, 1.0])
@pytest.mark.parametrize('dist', DISTS)
@pytest.mark.parametrize('K', SIZES)
def test_elite_exact_with_shards(eng, K, dist, pct):
    pos, neg = fitnesses(dist, K, 1, seed=K + 31 * DISTS.index(dist) + 7)
    inds = np.random.RandomState(K).randint(0, 10 ** 8, K).astype(np.int64)
    fp, fn, di = eng.to_device(pos), eng.to_device(neg), eng.to_device(inds)
    for name in SHAPINGS:
        with np.errstate(all='ignore'):
            vals, sel, fit, n_el = orc.elite_ranker(pos, neg, inds, name, pct)
        defined = not (name == 'max_normalized' and dist in ('pos_inf', 'outlier'))   # equal shaped values of distinct fitnesses
        out = eng.rank_transform(fp, fn, _kind(name), elite_n=n_el, noise_idx=di, want64=True, want_elite=True)
        _check_elite(out, vals, sel, fit, K, name, defined)
        dt = np.float64 if name == 'max_normalized' else np.float32
        pw = np.zeros(K, dtype=dt)
        for vv, f in zip(np.asarray(vals, dtype=dt), out['elite_fit'].cpu().numpy()):   # two terms at most: order-free
            pw[f % K] += vv
        assert _same(out['weights64'].cpu().numpy(), pw.astype(np.float64)), name
        if pct != 0.1:
            continue
        whole = {k: out[k].cpu().numpy() for k in ('elite_vals', 'elite_fit', 'elite_idx')}
        for N in (2, 3, 8):
            rebuilt = {k: np.zeros_like(v) for k, v in whole.items()}
            for b, cnt in _shards(K, N, K + N):
                part = eng.rank_transform(fp, fn, _kind(name), elite_n=n_el, k_begin=b, k_count=cnt, noise_idx=di, want64=True,
                                          want_elite=True)
                inside = (whole['elite_fit'] % K >= b) & (whole['elite_fit'] % K < b + cnt)
                for k, v in whole.items():
                    pv = part[k].cpu().numpy()
                    assert _same(pv[inside], v[inside]), (name, N, b, k)
                    assert not pv[~inside].any(), (name, N, b, k)
                    rebuilt[k][inside] = pv[inside]
                assert _same(part['weights64'].cpu().numpy(), out['weights64'].cpu().numpy()[b:b + cnt]), (name, N, b)
            for k, v in whole.items():
                assert _same(rebuilt[k], v), (name, N, k)


def test_reversed_elite_orders_ties_by_index(eng):
    """max_normalized with max + min < 0 (every reward negative): tied fitnesses inside the elite and a tie group across the
    threshold take the oracle's slots and members."""
    pos = np.array([[-3.], [-6.], [-6.], [-5.], [-6.], [-2.]])
    neg = np.array([[-6.], [-4.], [-2.], [-6.], [-1.], [-2.]])
    inds = np.arange(100, 106, dtype=np.int64)
    for pct in (0.25, 0.5, 1.0):                        # 3 of the five -6s; the five and the -5; everything (three -2s)
        vals, sel, fit, n_el = orc.elite_ranker(pos, neg, inds, 'max_normalized', pct)
        out = eng.rank_transform(eng.to_device(pos), eng.to_device(neg), _kind('max_normalized'), elite_n=n_el,
                                 noise_idx=eng.to_device(inds), want_elite=True)
        assert np.array_equal(out['elite_fit'].cpu().numpy(), fit), pct
        assert np.array_equal(out['elite_idx'].cpu().numpy(), sel), pct
        assert _same(out['elite_vals'].cpu().numpy(), np.asarray(vals, dtype=np.float64)), pct


def test_one_bucket_time_at_40000(eng):
    """The finalize is linear in its bucket's occupancy, so one outlier (every other value in one bucket) makes it quadratic:
    the time of one rank_transform at K = 40 000, printed with the device's name."""
    K = 40000
    pos, neg = fitnesses('outlier', K, 1, seed=5)
    fp, fn = eng.to_device(pos), eng.to_device(neg)
    for _ in range(3):
        eng.rank_transform(fp, fn, 0)
    eng.sync()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    reps = 10
    ev[0].record()
    for _ in range(reps):
        eng.rank_transform(fp, fn, 0)
    ev[1].record()
    eng.sync()
    ms = ev[0].elapsed_time(ev[1]) / reps
    pos_g, neg_g = fitnesses('gaussian', K, 1, seed=5)
    gp, gn = eng.to_device(pos_g), eng.to_device(neg_g)
    eng.rank_transform(gp, gn, 0)
    ev[0].record()
    for _ in range(reps):
        eng.rank_transform(gp, gn, 0)
    ev[1].record()
    eng.sync()
    ms_g = ev[0].elapsed_time(ev[1]) / reps
    print(f'\n[rank scale] K = {K}: one bucket {ms:.3f} ms, gaussian {ms_g:.3f} ms per rank_transform '
          f'on {torch.cuda.get_device_name(0)}')
