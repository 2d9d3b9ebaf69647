"""CPU checks of the unknown-scale stage's chunked sweep: the numpy restatement of the regenerating route equals the
restatement of the one-shot radix-sort route bit for bit at every chunk capacity, through split tie groups, partial
tiles carried between chunks, excluded measurements and an end point at +inf; and the two context calls that set and
report the chunking are declared, exported and bound."""
import importlib
import os
import re

import numpy as np
import pytest

import scale_stream_reference as ref

capi = importlib.import_module("teaser-plusplus_b200.capi")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(a, b):
    assert (np.isnan(a) and np.isnan(b)) or np.float64(a).tobytes() == np.float64(b).tobytes(), (a, b)


def _capacities(K):
    M = 2 * K
    return sorted({c for c in (2048, 2049, 3000, 4096, 6143, M // 3, M - 1, M, M + 5) if c >= 2048})


def _random(K, seed):
    rng = np.random.default_rng(seed)
    x = np.where(rng.random(K) < 0.3, rng.uniform(0.5, 3.0, K), 1.7 + rng.normal(0, 0.01, K))
    return x, rng.uniform(0.001, 0.05, K)


def _ties(K, seed):
    rng = np.random.default_rng(seed)
    return rng.choice([1.0, 1.5, 2.0, 1.25], K), rng.choice([0.25, 0.5, 0.125], K)


CASES = {
    "random": lambda: _random(5000, 1),
    "ties": lambda: _ties(4000, 2),
    "tiles_exact": lambda: _random(3 * 2048, 3),       # 2K a multiple of 2048
    "tiles_plus_one": lambda: _random(3 * 2048 + 1, 4),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_chunked_equals_one_shot(case):
    x, r = CASES[case]()
    want = ref.one_shot(x, r)
    assert np.isfinite(want)
    for C in _capacities(len(x)):
        _same(ref.chunked(x, r, C), want)


def test_tie_groups_split():
    x, r = _ties(4000, 2)
    key = np.sort(ref.keys(x, r), kind="stable")
    cuts = np.arange(2048, len(key), 2048)
    assert np.all(key[cuts - 1] == key[cuts])  # at C = 2048 every boundary falls inside a group of equal keys
    _same(ref.chunked(x, r, 2048), ref.one_shot(x, r))


def test_every_measurement_excluded():
    x = np.full(3000, np.inf)
    r = np.full(3000, np.inf)
    x[::2] = np.nan
    assert np.isnan(ref.one_shot(x, r))
    for C in (2048, 3000, 6000):
        assert np.isnan(ref.chunked(x, r, C))


def test_excluded_interleaved():
    x, r = _random(5000, 5)
    x[::3] = np.inf       # d1 = 0: ratio and range both infinite
    r[::3] = np.inf
    x[1::7] = np.nan      # d1 = d2 = 0
    r[1::7] = np.inf
    want = ref.one_shot(x, r)
    assert np.isfinite(want)
    for C in _capacities(len(x)):
        _same(ref.chunked(x, r, C), want)


def test_upper_end_point_at_infinity():
    x, r = _random(3000, 6)
    x[[11, 2501]] = 1.7e308   # kept (finite), but x + r rounds to +inf: tied with the excluded ones' keys, by q
    r[[11, 2501]] = 1e307
    x[::5] = np.inf
    r[::5] = np.inf
    assert np.isinf(x[11] + r[11]) and np.isfinite(x[11] - r[11])
    want = ref.one_shot(x, r)
    for C in _capacities(len(x)):
        _same(ref.chunked(x, r, C), want)


def test_radix_bits_order():
    v = np.array([-np.inf, -2.5, -1e-300, -0.0, 0.0, 1e-300, 1.0, 2.5, np.inf])
    b = ref.radix_bits(v)
    assert np.all(np.diff(b[[0, 1, 2, 3, 5, 6, 7, 8]].astype(object)) > 0) and b[3] == b[4]


SYMBOLS = {"tzr_ctx_set_scale_chunk": ["ctx", "max_end_points"], "tzr_ctx_last_scale_chunks": ["ctx"]}


@pytest.mark.parametrize("name", sorted(SYMBOLS))
def test_symbol_declared_and_bound(name):
    if not os.path.exists(capi.LIB_PATH):
        capi.build()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "teaser_b200.h")).read(), flags=re.S)
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)", hdr)
    assert m, f"{name} missing from the header"
    args = [a.split()[-1].lstrip("*") for a in " ".join(m.group(1).split()).split(",")]
    assert args == SYMBOLS[name]
    assert name in capi._SYMBOLS
    assert len(getattr(capi.lib(), name).argtypes) == len(args)


def test_calls_without_context():
    L = capi.lib()
    assert L.tzr_ctx_set_scale_chunk(None, 4096) == -1
    assert L.tzr_ctx_last_scale_chunks(None) == 0
