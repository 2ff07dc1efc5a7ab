"""GPU: the noise table drawn on the device (es_randn, Engine.randn, NoiseTable.make_noise_device / create_shared) against
numpy's legacy ``RandomState.randn``.

Equality criterion for a value: device float32 == numpy float32, or else it is one float32 ulp away AND numpy's float64 value
lies within 4 float64 ulps of the float32 rounding midpoint between the two (CUDA's log is not glibc's: the float64 gaussian
can differ in its last bit, which only shows after the float32 rounding next to a midpoint).  The stream state afterwards
(key, position, has_gauss) is bit-exact; the cached gaussian carries the same last-bit caveat."""
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch

from es_pytorch_b200.core.noisetable import NoiseTable

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _seeding():
    """The gym shim's seeding module, loaded by path (the shim directory is not put on sys.path here)."""
    path = os.path.join(ROOT, 'es_pytorch_b200', 'compat', 'gym', 'utils', 'seeding.py')
    spec = importlib.util.spec_from_file_location('_es_gym_seeding', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _state(rs):
    if rs == 'gym':
        return _seeding().np_random(4100, hashed=True)[0]
    return np.random.RandomState(rs)


def _upload(eng, rs):
    _, key, pos, has, gauss = rs.get_state()
    return [eng.to_device(np.asarray(key, dtype=np.uint32).view(np.int32)), eng.to_device(np.array([pos], dtype=np.int32)),
            eng.to_device(np.array([has], dtype=np.int32)), eng.to_device(np.array([gauss], dtype=np.float64))]


def _mismatches(got, ref64):
    """Asserts the equality criterion; returns the number of values that are not equal."""
    ref32 = ref64.astype(np.float32)
    assert got.shape == ref32.shape and got.dtype == np.float32
    bad = np.flatnonzero(got != ref32)
    if bad.size:
        g, r, r64 = got[bad], ref32[bad], ref64[bad]
        one_ulp = (g == np.nextafter(r, np.float32(np.inf))) | (g == np.nextafter(r, np.float32(-np.inf)))
        mid = (g.astype(np.float64) + r.astype(np.float64)) / 2
        near_mid = np.abs(r64 - mid) <= 4 * np.spacing(np.abs(r64))
        ok = one_ulp & near_mid
        assert ok.all(), [(int(i), float(a), float(b), float(c)) for i, a, b, c in zip(bad[~ok][:8], g[~ok], r[~ok], r64[~ok])]
    return int(bad.size)


def _assert_state(st_dev, rs):
    _, key, pos, has, gauss = rs.get_state()
    k, p, h, g = (t.cpu().numpy() for t in st_dev)
    assert np.array_equal(k.view(np.uint32), key), 'key'
    assert int(p[0]) == pos, ('pos', int(p[0]), pos)
    assert int(h[0]) == has, ('has_gauss', int(h[0]), has)
    assert abs(float(g[0]) - gauss) <= 2 * np.spacing(abs(gauss)), ('gauss', float(g[0]), gauss)


def _draw_and_check(eng, rs, n):
    st = _upload(eng, rs)
    got = eng.randn(*st, n)
    eng.sync()
    _mismatches(got.cpu().numpy(), rs.randn(n))
    _assert_state(st, rs)
    return got


@pytest.mark.parametrize('n', [0, 1, 2, 3, 623, 624, 625, 4 * 624 - 1, 4 * 624 + 1, 10 ** 6 + 1])
@pytest.mark.parametrize('seed', [0, 1, 12345, 2 ** 32 - 1, 'gym'])
def test_randn_matches_numpy_from_a_fresh_state(eng, seed, n):
    """A freshly seeded RandomState (position 624: the first draw regenerates the block), every size around the block
    length and an odd size past a million."""
    _draw_and_check(eng, _state(seed), n)


# words consumed before the draw: randint(0, 2**31) takes one word, random() two; randn(k) for odd k leaves a cached gaussian
_PREFIX = {
    'w1': lambda rs: rs.randint(0, 2 ** 31),
    'w2': lambda rs: rs.random(),
    'w3': lambda rs: (rs.randint(0, 2 ** 31), rs.random()),
    'w5': lambda rs: (rs.random(), rs.random(), rs.randint(0, 2 ** 31)),
    'g1': lambda rs: rs.randn(1),
    'g3': lambda rs: rs.randn(3),
    'w1g1': lambda rs: (rs.randint(0, 2 ** 31), rs.randn(1)),
    'w3g3': lambda rs: (rs.randint(0, 2 ** 31), rs.random(), rs.randn(3)),
    'block_end': lambda rs: rs.randint(0, 2 ** 31, size=624),
}


@pytest.mark.parametrize('n', [1, 2, 7, 100_000, 100_001])
@pytest.mark.parametrize('prefix', sorted(_PREFIX))
def test_randn_from_any_incoming_state(eng, prefix, n):
    """Attempts that start at every phase of the word grid, a pending cached gaussian (out[0]) and a position at the end of
    a block; then a second draw that continues from the state the first one left on the device."""
    rs = np.random.RandomState(777)
    _PREFIX[prefix](rs)
    st = _upload(eng, rs)
    for m in (n, n + 3):
        got = eng.randn(*st, m)
        eng.sync()
        _mismatches(got.cpu().numpy(), rs.randn(m))
        _assert_state(st, rs)


@pytest.mark.parametrize('blocks,jump_lb', [(64, None), (200, 2), (1, 0)])
def test_randn_window_edges(eng, monkeypatch, blocks, jump_lb):
    """Windows of a few blocks (dozens to thousands per draw): every window edge is crossed by attempts of every phase.
    The values and the end state are identical to the one-window draw and meet the criterion against numpy."""
    n = 2_000_001 if blocks > 1 else 200_001
    rs = np.random.RandomState(31337)
    rs.randint(0, 2 ** 31)
    rs.randn(1)
    one = _upload(eng, rs)
    want = eng.randn(*one, n)
    eng.sync()
    monkeypatch.setenv('ES_RANDN_WINDOW_BLOCKS', str(blocks))
    if jump_lb is not None:
        monkeypatch.setenv('ES_MT_JUMP_LB', str(jump_lb))
    _, windows = eng.randn_plan(n)
    assert windows >= 24, windows
    many = _upload(eng, rs)
    got = eng.randn(*many, n)
    eng.sync()
    assert torch.equal(got, want)
    for a, b in zip(many, one):
        assert torch.equal(a, b)
    _mismatches(got.cpu().numpy(), rs.randn(n))
    _assert_state(many, rs)


def test_randn_full_table_size(eng):
    """The shipped table: 250 000 000 values of one seed, compared with numpy chunk by chunk (numpy's chunked randn
    continues the same stream), and the end state."""
    n, chunk = 250_000_000, 10_000_000
    rs = np.random.RandomState(2024)
    st = _upload(eng, rs)
    got = eng.randn(*st, n)
    eng.sync()
    bad = 0
    for lo in range(0, n, chunk):
        bad += _mismatches(got[lo:lo + chunk].cpu().numpy(), rs.randn(chunk))
    print(f'250 M values: {bad} differ by one float32 ulp next to a rounding midpoint')
    assert bad <= 8, bad
    _assert_state(st, rs)


def test_make_noise_device_is_deterministic(eng):
    a = NoiseTable.make_noise_device(1_000_003, 99, engine=eng)
    b = NoiseTable.make_noise_device(1_000_003, 99, engine=eng)
    assert a.device == eng.device and a.dtype == torch.float32 and a.shape == (1_000_003,)
    assert torch.equal(a, b)
    _mismatches(a.cpu().numpy(), np.random.RandomState(99).randn(1_000_003))


def test_make_noise_device_gym_seeding(eng, monkeypatch):
    """gym_seeding=True seeds the host RandomState through gym.utils.seeding like make_noise (here the shim's)."""
    gym, utils = types.ModuleType('gym'), types.ModuleType('gym.utils')
    utils.seeding = _seeding()
    gym.utils = utils
    monkeypatch.setitem(sys.modules, 'gym', gym)
    monkeypatch.setitem(sys.modules, 'gym.utils', utils)
    got = NoiseTable.make_noise_device(50_001, 4100, gym_seeding=True, engine=eng).cpu().numpy()
    want = NoiseTable.make_noise(50_001, 4100, gym_seeding=True)
    ref64 = _state('gym').randn(50_001)
    assert np.array_equal(want, ref64.astype(np.float32)) and not np.array_equal(want, NoiseTable.make_noise(50_001, 4100))
    _mismatches(got, ref64)


class _Comm:
    rank, size = 0, 1


def test_create_shared_builds_the_table_on_the_device(eng, monkeypatch):
    monkeypatch.delenv('ES_NOISE_TABLE_HOST', raising=False)
    nt = NoiseTable.create_shared(_Comm(), 300_001, 100, None, [5])
    assert nt._host is None, 'no host table is built'
    dev = nt.device_table(eng)
    assert dev.is_cuda and dev.dtype == torch.float32 and len(nt) == 300_001
    assert torch.equal(dev, NoiseTable.make_noise_device(300_001, 5, engine=eng))
    host = nt.noise
    assert np.array_equal(host, dev.cpu().numpy())
    assert np.array_equal(nt.get(17, 100), host[17:117])
    _mismatches(host, np.random.RandomState(5).randn(300_001))


def test_create_shared_host_path_on_request(eng, monkeypatch):
    monkeypatch.setenv('ES_NOISE_TABLE_HOST', '1')
    nt = NoiseTable.create_shared(_Comm(), 300_001, 100, None, 5)
    assert nt._dev is None and np.array_equal(nt.noise, np.random.RandomState(5).randn(300_001).astype(np.float32))
    assert np.array_equal(nt.device_table(eng).cpu().numpy(), nt.noise)


def test_randn_rejects_bad_arguments(eng):
    st = _upload(eng, np.random.RandomState(0))
    with pytest.raises(ValueError):
        eng.randn(*st, -1)
    with pytest.raises(TypeError):
        eng.randn(st[0].to(torch.int64), *st[1:], 10)
    assert eng.randn(*st, 0).numel() == 0
    assert eng.randn_plan(0) == (0, 0)
    nbytes, windows = eng.randn_plan(250_000_000)
    assert windows > 1 and nbytes <= 320 * 2 ** 20, (nbytes, windows)
