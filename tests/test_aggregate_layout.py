"""Pins, per way an aggregate's buffers can be laid out (function family x how the slots hold the value), the generated
source of a plan and the bytes sd_partial_merge / sd_final_merge return for a seeded stream of partial rows from several
partitions.  The stream carries NULL buffers, empty groups (the buffers before any input), wide-DECIMAL sums past the
buffer's precision and NaNs.  Host only: no device is needed."""
import ctypes as C
import hashlib
import random
import struct

import pytest

from snappydata_b200 import capi
from snappydata_b200.capi import MOMENT_BUFFERS, ORDER_AGGS, PAIR_BUFFERS, AggFn
from snappydata_b200.column_format import SqlType as T, unsafe_row
from snappydata_b200.plan import PlanBuilder
from test_moment_aggregates import _codegen


def _cols(b):
    return {
        "l": b.col(T.LONG, 1, True),
        "d": b.col(T.DOUBLE, 2, True),
        "i": b.col(T.INT, 3, True),
        "s": b.col(T.STRING, 4, True),
        "m": b.col(T.DECIMAL, 5, True, scale=2, precision=15),
        "w": b.col(T.DECIMAL, 6, True, scale=2, precision=38),
        "y": b.col(T.DOUBLE, 7, True),
    }


def _count(b, c): b.count().count(c["l"]).count(c["s"])
def _sum_word(b, c): b.sum(c["l"]).sum(c["d"]).avg(c["d"]).avg(c["l"])
def _dec15(b, c): b.sum(c["m"]).avg(c["m"])
def _dec38(b, c): b.sum(c["w"]).avg(c["w"])
def _minmax(b, c): b.min(c["i"]).max(c["d"]).min(c["m"]).max(c["l"]).min(c["s"]).max(c["s"]).min(c["w"]).max(c["w"])
def _moments(b, c): b.stddev_pop(c["d"]).stddev_samp(c["d"]).var_pop(c["d"]).var_samp(c["d"]).skewness(c["d"]).kurtosis(c["d"])
def _pairs(b, c): b.covar_pop(c["d"], c["y"]).covar_samp(c["d"], c["y"]).corr(c["d"], c["y"])


def _first_last(b, c):
    for n in ("d", "s", "w"):
        b.first(c[n]).last(c[n]).first(c[n], ignore_nulls=True).last(c[n], ignore_nulls=True)


AGGS = {"count": _count, "sum_word": _sum_word, "dec15": _dec15, "dec38": _dec38, "minmax": _minmax, "moments": _moments,
        "pairs": _pairs, "first_last": _first_last}


def _plan(aggs, keys):
    b = PlanBuilder()
    k0, k1 = b.col(T.STRING, 0, True), b.col(T.LONG, 8, True)
    c = _cols(b)
    if keys == "keyed":
        b.group_by(k0, k1)
    elif keys == "rollup":
        b.rollup(k0, k1)
    AGGS[aggs](b, c)
    return b.build()


PLANS = [(a, k) for a in AGGS for k in ("keyed", "nokey")] + [("moments", "rollup"), ("first_last", "rollup"), ("dec38", "rollup")]

# ---- a seeded partial-row stream ------------------------------------------------------------------------------------------


def _dec(rng, p):
    lim = 10 ** p
    r = rng.random()
    if r < 0.2:
        return rng.choice([1, -1]) * (lim - rng.randrange(1, 1000))   # near the bound: sums of two pass it
    if r < 0.25 and p == 38:
        return lim   # a wide sum that overflowed in its partition
    return rng.randrange(-10 ** min(p, 12), 10 ** min(p, 12))


def _value(rng, t, nullable=True):
    if nullable and rng.random() < 0.12:
        return None
    if isinstance(t, tuple):
        return _dec(rng, t[1])
    if t == T.DOUBLE:
        return rng.choice([float("nan"), -0.0, 0.0, rng.uniform(-1e3, 1e3), rng.uniform(-1e3, 1e3), float(rng.randrange(0, 40))])
    if t == T.STRING:
        return rng.choice(["", "a", "ab", "b", "zzé", "abcdefghijklmnopq"])
    if t == T.BOOLEAN:
        return rng.random() < 0.6
    if t == T.INT:
        return rng.randrange(-1000, 1000)
    return rng.randrange(-(1 << 40), 1 << 40)


def _width(fn):
    if fn == AggFn.AVG or fn in ORDER_AGGS:
        return 2
    return MOMENT_BUFFERS.get(fn) or PAIR_BUFFERS.get(fn) or 1


def _buffers(rng, fn, types):
    """one aggregate's partial buffer: an empty one (before any input) or a seeded one, NULLs where Spark has them"""
    if rng.random() < 0.15:   # empty
        if fn in (AggFn.COUNT_STAR, AggFn.COUNT):
            return [0]
        if fn == AggFn.AVG:
            return [0 if isinstance(types[0], tuple) else 0.0, 0]
        if fn in ORDER_AGGS:
            return [None, False]
        if fn in MOMENT_BUFFERS or fn in PAIR_BUFFERS:
            return [0.0] * len(types)
        return [None]
    if fn in (AggFn.COUNT_STAR, AggFn.COUNT):
        return [rng.randrange(0, 1000)]
    if fn == AggFn.AVG:
        return [_value(rng, types[0], False), rng.randrange(1, 50)]
    if fn in ORDER_AGGS:
        return [_value(rng, types[0]), True]
    if fn in MOMENT_BUFFERS or fn in PAIR_BUFFERS:
        return [float(rng.randrange(1, 30))] + [_value(rng, T.DOUBLE, False) for _ in types[1:]]
    return [_value(rng, types[0])]


def _stream(desc, seed, partitions=4, rows=40):
    rng = random.Random(seed)
    schema = desc.partial_schema()
    nk = len(desc.keys_py)
    out = b""
    for _ in range(partitions):
        for _ in range(rows):
            vals = [rng.choice([None, "a", "bb", "c"]) if t == T.STRING else rng.choice([None, 1, 2, -7]) for t in schema[:nk]]
            if desc.keys_py and schema[nk - 1] == T.INT and len(desc.keys_py) == 3:   # ROLLUP (k0, k1): spark_grouping_id
                vals[-1] = rng.choice([0, 1, 3])
            k = nk
            for fn, _ in desc.aggs_py:
                w = _width(fn)
                vals += _buffers(rng, fn, schema[k:k + w])
                k += w
            row = unsafe_row(list(zip(schema, vals)))
            out += struct.pack("<q", len(row)) + row
    return out


def _merge(fn, desc, raw):
    cap = max(1 << 16, 4 * len(raw) + 1024)
    buf = C.create_string_buffer(cap)
    out_len, out_rows = C.c_int64(), C.c_int64()
    api = capi.product_api()
    api.check(fn(C.byref(desc.c), capi._buf_ptr(raw), len(raw), buf, cap, C.byref(out_len), C.byref(out_rows)))
    return buf.raw[: out_len.value] + struct.pack("<q", out_rows.value)


def _digest(desc):
    api = capi.product_api()
    h = hashlib.sha256()
    for seed in (1, 2, 3):
        raw = _stream(desc, seed)
        h.update(_merge(api.partial_merge, desc, raw))
        h.update(_merge(api.final_merge, desc, raw))
    h.update(_merge(api.partial_merge, desc, b""))   # no partitions: the no-key row of empty buffers
    h.update(_merge(api.final_merge, desc, b""))
    return h.hexdigest()


# sha256 of (generated source, merge outputs) at the commit before aggregate layouts were recorded in plan analysis
PINNED = {
    "count-keyed": ("ac9f75410d18af098e7bd99963c7005555f4825102989d2d069aa8f9d55f31f1",
        "2ad85cd2808d9c7f0c507c09fd21c27704bd48d1854b88741bdb3f3de71e6a00"),
    "count-nokey": ("ace25969f3927e434a412f7cfd1de707a9ce9419b0f135fed1e5d36a3861348e",
        "714206f16038746a397c7271435ce967ec73c4618cb4c3033f7d2a88904c66be"),
    "sum_word-keyed": ("0bc2fe90962c4d31e4ba20811fa1e0ede04447a9b3bc68c2d68f7bdcd21e7000",
        "575204a06938d9bad170ca82f154921aed56669e1f60c7f0cd6f8b7679d7a709"),
    "sum_word-nokey": ("af3cf1628d4c4c3cc3ef28aaa903bc5207fe677fc23bb0b39384097b9a879bb6",
        "56844105a06346a99e091b1e8911b340c739ef8a15541a99f7b6871e59b582e6"),
    "dec15-keyed": ("74ec9b556d178708e64f7adfd9099746fece829488ae48b68d8602b496ca3544",
        "7e05fe95ac80d5e0a2a2db14cd609c6ac45159a13c634490e74e3ef88b4152b9"),
    "dec15-nokey": ("b0be51856468553a76be6a4bc871a29d12072d6a8a283c283b17643ca9cb0461",
        "25ac3c61dd623ce2d07a57afd7eaeb5805f12927158a5043530c1456e300608a"),
    "dec38-keyed": ("825281663bb26f1398be77fe71666bcbf54c76e4e4a97455609280e78cd41361",
        "962623e5c630ddca4b80d60de065cc1ed5d6c125353f241d6a025a006992e9e6"),
    "dec38-nokey": ("7d8cda157ab502e9cc22e851bbc3f41790feb348154a07f4c885ea0ac569174b",
        "c764713a6f14c526968f2107bd285447a7727e4626f8b9f3a541daf28f8145c6"),
    "minmax-keyed": ("7c500f9acc72c73541b5707f0009a936ecd9749562c053f45e6c235c9be826c7",
        "5f6bad162c5753b6f21901b51e0bbfcf1d7fc6471f7f1fbeb140de91162dff4b"),
    "minmax-nokey": ("a4e1b8d86e0de24193424abfb711735723ff2ad42dbbf14fc2a13af6e4220f94",
        "5b6c8b62de817c6ba291d8303dfed45a90e3b1856dbc4028ed5f778a9afb4946"),
    "moments-keyed": ("3dc0a80eebd617395fed14af4e19e9ceb0ea70310f75b5cb67a7910cfb4e85bc",
        "b15ba753515ba018bb5c8e96b28651193a83764362bd970c0714edbdff7966ac"),
    "moments-nokey": ("700b4df1d673cbb2b103099bdd6625935e4307214cb8a2ba3084643d208940cd",
        "074b25ebcdeb1a3867fb2bcb7de5eb017ad2ffed1d3dbfe167aa892466508ac9"),
    "pairs-keyed": ("4c2fd2c29f3678c465c58770781a2b334a3df8ab271ed89e1fd878d82edc8de0",
        "a0d965657e437b8527a07c4c6d65e62c595e84359fb03ea6e73ac05829208cac"),
    "pairs-nokey": ("4e9c9e3996c5909ff19462e31a2128de8416c635238634d2205a53446c57537d",
        "9909e1d6f97aa35a07ab5f0fef0ea8fec1487fe18c87de37e5e77765c8d2152d"),
    "first_last-keyed": ("f8fb036bb17a744ee084f7abbad7993a1c9b0f138a47cc67c47407bd0c5b7ac4",
        "5aa02a0be6672226c1a86c2af1dc89e252b1808a2230af481f211bc40c51406b"),
    "first_last-nokey": ("cce36da559563531f5238de15373fbff90e9e7c58ffba7c9ad0fdea355ae3b2f",
        "eea819ac213024422706fff508a022eba07da29cc988c111e05826bed50c436b"),
    "moments-rollup": ("3dc0a80eebd617395fed14af4e19e9ceb0ea70310f75b5cb67a7910cfb4e85bc",
        "49aedf2e0433e928f490b0872eddb0e828385edea097ad345bacd1d887da51a6"),
    "first_last-rollup": ("f8fb036bb17a744ee084f7abbad7993a1c9b0f138a47cc67c47407bd0c5b7ac4",
        "58d7085ad6e65fbc4dc4bf8668b9647ca841ffc69e6c7891feb39c4cab4122ad"),
    "dec38-rollup": ("825281663bb26f1398be77fe71666bcbf54c76e4e4a97455609280e78cd41361",
        "ef999831f7379d135abb256cf0ff5bf0d1d85ae22ca2fb44880433310ae9b58c"),
}


@pytest.mark.parametrize("aggs,keys", PLANS, ids=[f"{a}-{k}" for a, k in PLANS])
def test_generated_source_and_host_merges_are_pinned(aggs, keys):
    desc = _plan(aggs, keys)
    rc, src, _ = _codegen(desc)
    assert rc == 0, src
    got = (hashlib.sha256(src.encode()).hexdigest(), _digest(desc))
    assert got == PINNED[f"{aggs}-{keys}"]


def test_merge_errors_keep_their_codes_and_messages():
    api = capi.product_api()
    desc = _plan("sum_word", "keyed")
    raw = _stream(desc, 1, partitions=1, rows=2)
    bad = bytearray(raw[:16])
    struct.pack_into("<q", bad, 0, 8)   # a row too short for its fields
    b = PlanBuilder()
    b.project(b.col(T.LONG, 0, True))
    cases = [(api.final_merge, desc, raw[:-3], "sd_final_merge: bad row size"),
             (api.partial_merge, desc, bytes(bad), "sd_final_merge: malformed partial row"),
             (api.final_merge, b.build(), raw[:-3], "merge: bad row size")]
    for fn, d, stream, msg in cases:
        with pytest.raises(capi.SdError) as e:
            _merge(fn, d, stream)
        assert e.value.code == capi.SD_ERR_INVALID and str(e.value).endswith(msg), str(e.value)


def _half_up(num, den):
    q, r = divmod(abs(num), den)
    return (1 if num >= 0 else -1) * (q + (2 * r >= den))


@pytest.mark.parametrize("aggs,big", [("dec15", 10 ** 14 + 1), ("dec38", 10 ** 33 + 1)])
def test_decimal_avg_rounds_half_up_at_ties(aggs, big):
    """AVG over DECIMAL(p,2) is DECIMAL(p+4,6): sum * 10^4 / count, HALF_UP.  An odd sum over 32 rows lands exactly halfway,
    so rounding half down or half even would change the last digit; each group is two partitions of 16 rows"""
    desc = _plan(aggs, "keyed")
    schema = desc.partial_schema()   # keys ++ SUM ++ AVG [sum, count]
    sums = {"a": 1, "b": -1, "c": 3, "bb": -big}
    raw = b""
    for key, s in sums.items():
        for part in (s // 2, s - s // 2):
            row = unsafe_row(list(zip(schema, [key, 1, part, part, 16])))
            raw += struct.pack("<q", len(row)) + row
    got = {r[0].decode(): r[3] for r in capi.final_merge(capi.product_api(), desc, raw)}
    assert got == {k: _half_up(s * 10 ** 4, 32) for k, s in sums.items()}
    assert all(s * 10 ** 4 % 32 == 16 for s in sums.values())
