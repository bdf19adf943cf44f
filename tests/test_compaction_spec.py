"""The two definitions of a compacted (folded) column pinned against each other on the host, without a GPU: the reference's
ColumnDeltaEncoder.merge into a full column (sd_delta_merge with existing_is_delta = 0, depth-1 delta first, then depth 0)
and the fixture writer's default encoder over the effective values (what sd_store_encode_batch writes and sd_store_compact
must write).  Every fixed-width type and STRING, nullable and NOT NULL, random bases and deltas."""
import ctypes as C

import numpy as np
import pytest

from snappydata_b200 import capi
from snappydata_b200.column_format import SqlType as T, encode_column, encode_delta

TYPES = [T.BYTE, T.SHORT, T.INT, T.DATE, T.LONG, T.TIMESTAMP, T.DECIMAL, T.FLOAT, T.DOUBLE, T.BOOLEAN, T.STRING]


def _fold(t, nullable, delta, column, num_rows):
    api = capi.product_api()
    f = api.lib.sd_delta_merge
    f.restype = C.c_int
    f.argtypes = [C.POINTER(capi.sd_column), C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int32, C.c_int32, C.c_char_p, C.c_int64,
                  C.POINTER(C.c_int64)]
    col = capi.sd_column(int(t), int(nullable), 0, 0, 18 if t == T.DECIMAL else 0)
    out = C.create_string_buffer(len(delta) + len(column) + 4096)
    n = C.c_int64()
    api.check(f(C.byref(col), delta, len(delta), column, len(column), 0, num_rows, out, len(out), C.byref(n)))
    return out.raw[: n.value]


def _values(t, r, m):
    if t == T.STRING:
        return np.array([b"s%d" % x for x in r.integers(0, 40, m)], dtype=object)
    if t == T.BOOLEAN:
        return r.integers(0, 2, m).astype(bool)
    if t in (T.DOUBLE, T.FLOAT):
        return np.round(r.normal(0, 50, m), 2).astype("<f8" if t == T.DOUBLE else "<f4")
    lo, hi = {T.BYTE: (-128, 128), T.SHORT: (-2000, 2000)}.get(t, (-10**6, 10**6))
    return r.integers(lo, hi, m)


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("seed", [1, 2])
def test_host_fold_equals_the_default_encoder_over_the_effective_values(t, nullable, seed):
    r = np.random.default_rng(seed * 100 + int(t) * 2 + nullable)
    n = 3000 if seed == 1 else 777
    base = _values(t, r, n)
    eff = list(base) if t == T.STRING else base.copy()
    base_nulls = (r.random(n) < 0.15) if nullable else None
    eff_nulls = base_nulls.copy() if nullable else np.zeros(n, bool)
    col = encode_column(base, t, base_nulls)
    for depth in (1, 0):   # the older delta is folded first; depth 0 wins where both hold a position
        m = int(r.integers(1, n // 4))
        pos = np.sort(r.choice(n, m, replace=False)).astype(np.int32)
        if depth == 0 and seed == 1:   # also overwrite rows the depth-1 delta already holds
            pos = np.unique(np.concatenate([pos, pos[: m // 3]])).astype(np.int32)
        vals = _values(t, r, len(pos))
        dn = (r.random(len(pos)) < 0.2) if nullable else None
        col = _fold(t, nullable, encode_delta(n, pos, vals, t, dn), col, n)
        for k, p in enumerate(pos):
            eff[p] = vals[k]
        if nullable:
            eff_nulls[pos] = dn
    want = encode_column(np.array(eff, dtype=object) if t == T.STRING else eff, t, eff_nulls if nullable else None)
    assert col == want


@pytest.mark.parametrize("t", [T.INT, T.STRING, T.DOUBLE])
def test_fold_that_clears_every_null_trims_the_null_words(t):
    r = np.random.default_rng(5)
    n = 500
    base, nulls = _values(t, r, n), np.zeros(n, bool)
    nulls[[3, 70, 300]] = True
    col = encode_column(base, t, nulls)
    pos = np.array([3, 70, 300], np.int32)
    vals = _values(t, r, 3)
    got = _fold(t, True, encode_delta(n, pos, vals, t), col, n)
    eff = np.array(list(base), dtype=object) if t == T.STRING else base.copy()
    eff[pos] = vals
    assert got == encode_column(eff, t, None) == encode_column(eff, t, np.zeros(n, bool))
