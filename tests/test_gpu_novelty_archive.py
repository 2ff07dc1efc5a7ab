"""es_novelty bit for bit against orc.novelty (novelty.py:16-18) at grown archives: NSRA appends a behaviour every generation, so
the archive runs from 1 entry to thousands.  k up to the kernel's 64, k larger than the archive (heapq.nsmallest clips it),
duplicate archive rows, a behaviour on an archive row (distance 0), and 20 000 evaluations written with a stride of 2.

Both sides take the k smallest correctly rounded float64 distances in ascending order; the mean is np.mean's, whose sum is
numpy's pairwise summation (eight interleaved partial sums from 8 terms on), not a left-to-right sum.
"""
import numpy as np
import pytest
import torch

from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu


def _case(rs, n, A, dup):
    behv = (rs.randn(n, 3) * 3).astype(np.float32)
    archive = rs.randn(A, 2) * 3
    if dup and A > 2:
        archive[1::2] = archive[0:A - 1:2][:len(archive[1::2])]        # every other row repeats the one before it
    if A >= 1 and n >= 2:
        behv[1, :2] = archive[A // 2]                                   # float32 copy: distance 0 only if it rounds back
        archive[A // 2] = behv[1, :2].astype(np.float64)
    return behv, archive


def _novelty(eng, behv, archive, k, stride=1):
    n = len(behv)
    out = torch.full((n * stride,), -1.0, dtype=torch.float64, device=eng.device)
    eng.novelty(eng.to_device(behv), eng.to_device(archive), k, out, stride)
    eng.sync()
    return out.cpu().numpy()


@pytest.mark.parametrize('dup', [False, True])
@pytest.mark.parametrize('A', [1, 63, 64, 65, 1000, 5000])
def test_novelty_bit_exact_at_grown_archives(eng, A, dup):
    rs = np.random.RandomState(A + 7 * dup)
    behv, archive = _case(rs, 300, A, dup)
    for k in (1, 10, 63, 64):
        got = _novelty(eng, behv, archive, k)
        ref = np.array([orc.novelty(behv[i, :2], archive, k) for i in range(len(behv))])
        bad = np.flatnonzero(got != ref)
        assert bad.size == 0, (A, k, bad[:5], got[bad[:3]], ref[bad[:3]])


def test_novelty_20000_evaluations_strided(eng):
    rs = np.random.RandomState(3)
    behv, archive = _case(rs, 20000, 64, True)
    got = _novelty(eng, behv, archive, 10, stride=2)
    ref = np.array([orc.novelty(behv[i, :2], archive, 10) for i in range(len(behv))])
    assert np.array_equal(got[0::2], ref)
    assert np.all(got[1::2] == -1.0)                                    # the stride's gaps are not written
