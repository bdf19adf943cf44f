"""Host-only checks of GROUP BY ... WITH ROLLUP / WITH CUBE / GROUPING SETS: the reference's closed forms on the CPU oracle
(Expand restated per set, tests/grouping_sets_cases.py) with the product's host final merge of the same partial rows, the
scan kernel's generated source being the plain GROUP BY's, every refusal of the GROUPING_SET / GROUPING_ID nodes, and gid as a
merge key."""
import ctypes as C
import struct

import pytest

import grouping_sets_cases as G
import known_answer_cases as K
from oracle import oracle
from snappydata_b200 import build, capi
from snappydata_b200.capi import SD_PLAN_MUTATE, AggFn, Op, PlanDesc
from snappydata_b200.column_format import SqlType as T, parse_row_stream, unsafe_row
from snappydata_b200.plan import PlanBuilder, q1_plan

SD_ERR_INVALID, SD_ERR_UNSUPPORTED = 1, 2


def _codegen(desc):
    lib = C.CDLL(build.build_codegen_lib())
    lib.sd_plan_codegen.restype = C.c_int
    lib.sd_plan_codegen.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.POINTER(C.c_int64), C.c_char_p, C.c_int64, C.c_char_p,
                                    C.c_int64, C.c_int32, C.c_int32, C.c_int32]
    src, sig, name, ln = C.create_string_buffer(1 << 18), C.create_string_buffer(1 << 16), C.create_string_buffer(256), C.c_int64()
    rc = lib.sd_plan_codegen(C.byref(desc.c), src, len(src), C.byref(ln), sig, len(sig), name, len(name), 0, 0, 0)
    return rc, src.value.decode(errors="replace"), sig.value.decode(errors="replace")


def _with_nodes(desc: PlanDesc, extra_nodes, keys=None, aggs=None, proj=None, flags=None, filter_node=None):
    return PlanDesc(desc.cols_py, desc.exprs_py + list(extra_nodes), desc.filter if filter_node is None else filter_node,
                    desc.keys_py if keys is None else keys, desc.aggs_py if aggs is None else aggs,
                    desc.proj_py if proj is None else proj, desc.literal_types_py, desc.flags if flags is None else flags)


# ---- closed forms ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", G.CLOSED_FORMS, ids=lambda c: c.__name__)
def test_closed_form_on_oracle_and_host_merge(case, oracle_api):
    eng = K.OracleEngine(oracle_api)

    def run(desc, lits, batches):
        rows = G.expand_reference(eng, desc, lits, batches)

        def partial_raw(sp, lits_, batches_):
            pl = oracle.plan(sp).set_literals(lits_)
            for b in batches_:
                pl.submit(b)
            return pl.finish_raw()
        raw = G.expand_partials(partial_raw, desc, lits, batches)
        product = capi.final_merge(capi.product_api(), desc, raw)
        assert sorted(map(repr, product)) == sorted(map(repr, rows))
        return rows, None
    case(run)


def test_rollup_and_cube_masks_follow_snappy_parser():
    b = PlanBuilder()
    k = [b.col(T.INT, i, True) for i in range(3)]
    b.rollup(*k).count()
    assert G.split(b.build())[1] == [0, 1, 3, 7]
    b.cube(*k)
    assert G.split(b.build())[1] == list(range(8))
    b.grouping_sets(k, [[k[0], k[2]], [k[1]], []])
    assert G.split(b.build())[1] == [0b010, 0b101, 0b111]


# ---- the scan is the plain GROUP BY's -------------------------------------------------------------------------------------
def _plain(desc):
    keys, _, first = G.split(desc)
    return PlanDesc(desc.cols_py, desc.exprs_py[:first], desc.filter, keys, desc.aggs_py, desc.proj_py, desc.literal_types_py)


def _q1_rollup():
    d = q1_plan()
    b_nodes = [(Op.GROUPING_SET, int(T.INT), m, 0, 0) for m in (0, 1, 3)]
    first = len(d.exprs_py)
    return _with_nodes(d, b_nodes + [(Op.GROUPING_ID, int(T.INT), first, 3, 0)], keys=d.keys_py + [first + 3])


def _hash_rollup():
    b = PlanBuilder()
    k1, k2, v = b.col(T.LONG, 0, True), b.col(T.DATE, 1, False), b.col(T.DOUBLE, 2, True)
    return b.rollup(k1, k2).sum(v).min(v).count().build()


def _moment_cube():
    b = PlanBuilder()
    k1, k2, x, y = b.col(T.STRING, 0, False), b.col(T.INT, 1, True), b.col(T.DOUBLE, 2, True), b.col(T.DOUBLE, 3, True)
    return b.cube(k1, k2).kurtosis(x).corr(x, y).build()


@pytest.mark.parametrize("make", [_q1_rollup, _hash_rollup, _moment_cube], ids=["q1", "hash", "moments"])
def test_generated_scan_is_the_plain_group_by(make):
    desc = make()
    rc, src, sig = _codegen(desc)
    rc0, src0, sig0 = _codegen(_plain(desc))
    assert rc == 0 and rc0 == 0, (src, src0)
    assert src == src0 and sig == sig0


def test_partial_and_final_schemas_carry_gid():
    desc = G.mytable_plan("cube")
    assert desc.partial_schema() == [T.INT, T.INT, T.INT, T.LONG]
    assert desc.final_schema() == [T.INT, T.INT, T.INT, T.LONG]


# ---- refusals ---------------------------------------------------------------------------------------------------------------
def _base():
    b = PlanBuilder()
    k1, k2, v = b.col(T.INT, 0, True), b.col(T.INT, 1, True), b.col(T.LONG, 2, True)
    b.group_by(k1, k2).sum(v)
    return b.build()


def _gs(masks, first):
    return [(Op.GROUPING_SET, int(T.INT), m, 0, 0) for m in masks] + [(Op.GROUPING_ID, int(T.INT), first, len(masks), 0)]


def _refusals():
    d = _base()
    n0 = len(d.exprs_py)
    gid = n0 + 2
    ok_nodes = _gs([0, 3], n0)
    yield "ok", _with_nodes(d, ok_nodes, keys=d.keys_py + [gid]), 0
    yield "set node outside a list", _with_nodes(d, [(Op.GROUPING_SET, int(T.INT), 0, 0, 0)]), SD_ERR_INVALID
    yield "gid not the last key", _with_nodes(d, ok_nodes, keys=[gid] + d.keys_py), SD_ERR_INVALID
    yield "gid not a key at all", _with_nodes(d, ok_nodes), SD_ERR_INVALID
    yield "set node as a key", _with_nodes(d, ok_nodes, keys=d.keys_py + [n0]), SD_ERR_INVALID
    yield "gid in a filter", _with_nodes(d, ok_nodes, keys=d.keys_py + [gid], filter_node=gid), SD_ERR_INVALID
    yield "gid as an operand", _with_nodes(d, ok_nodes + [(Op.ISNULL, int(T.BOOLEAN), gid, 0, 0)], keys=d.keys_py + [gid],
                                           filter_node=gid + 1), SD_ERR_INVALID
    yield "gid as an aggregate input", _with_nodes(d, ok_nodes, keys=d.keys_py + [gid], aggs=[(AggFn.SUM, gid)]), SD_ERR_INVALID
    yield "gid projected", _with_nodes(d, ok_nodes, keys=[], aggs=[], proj=[gid]), SD_ERR_INVALID
    yield "gid as a SET value", _with_nodes(d, ok_nodes, keys=[], aggs=[], proj=[gid], flags=SD_PLAN_MUTATE), SD_ERR_INVALID
    yield "mask bit at n", _with_nodes(d, _gs([0, 4], n0), keys=d.keys_py + [gid]), SD_ERR_INVALID
    yield "negative mask", _with_nodes(d, _gs([0, -1], n0), keys=d.keys_py + [gid]), SD_ERR_INVALID
    yield "no sets", _with_nodes(d, [(Op.GROUPING_ID, int(T.INT), n0, 0, 0)], keys=d.keys_py + [n0]), SD_ERR_INVALID
    yield "no GROUP BY expression", _with_nodes(d, _gs([0], n0), keys=[n0 + 1]), SD_ERR_UNSUPPORTED
    yield "duplicate masks", _with_nodes(d, _gs([1, 1], n0), keys=d.keys_py + [gid]), SD_ERR_UNSUPPORTED
    yield "gid in an UPDATE plan", _with_nodes(d, ok_nodes, keys=d.keys_py + [gid], aggs=[], flags=SD_PLAN_MUTATE), SD_ERR_UNSUPPORTED
    yield "gid in a projection plan", _with_nodes(d, ok_nodes, keys=[gid], aggs=[], proj=[0]), SD_ERR_UNSUPPORTED
    many = [(Op.GROUPING_SET, int(T.INT), m, 0, 0) for m in range(4097)]
    yield "more than 4096 sets", _with_nodes(d, many + [(Op.GROUPING_ID, int(T.INT), n0, 4097, 0)], keys=d.keys_py + [n0 + 4097]), SD_ERR_UNSUPPORTED
    b = PlanBuilder()
    ks = [b.col(T.INT, i, True) for i in range(32)]
    b.rollup(*ks).count()
    yield "32 GROUP BY expressions", b.build(), SD_ERR_UNSUPPORTED


@pytest.mark.parametrize("what,desc,status", list(_refusals()), ids=[r[0] for r in _refusals()])
def test_refusals(what, desc, status):
    rc, msg, _ = _codegen(desc)
    assert rc == status, (what, msg)


# ---- gid is a merge key ------------------------------------------------------------------------------------------------------
def _row(schema, vals):
    r = unsafe_row(list(zip(schema, vals)))
    return struct.pack("<q", len(r)) + r


def test_host_merges_by_keys_and_gid():
    desc = G.mytable_plan("cube")
    ps = desc.partial_schema()
    part1 = _row(ps, [1, None, 1, 10]) + _row(ps, [None, None, 3, 5]) + _row(ps, [1, None, 0, 7])   # (1, NULL) gid 1 vs a data NULL
    part2 = _row(ps, [1, None, 1, 20]) + _row(ps, [None, None, 3, 6])
    api = capi.product_api()
    got = sorted(capi.final_merge(api, desc, part1 + part2), key=repr)
    assert got == sorted([[1, None, 1, 30], [None, None, 3, 11], [1, None, 0, 7]], key=repr)
    merged = parse_row_stream(capi.partial_merge_raw(api, desc, part1 + part2), ps)
    assert sorted(merged, key=repr) == got


def test_more_than_16_shifts_refused_by_every_entry_point():
    b = PlanBuilder()
    k = b.col(T.INT, 0, True)
    xs = [b.col(T.DOUBLE, 1 + i, True) for i in range(17)]
    b.rollup(k)
    for x in xs:
        b.var_samp(x)
    desc = b.build()
    rc, msg, _ = _codegen(desc)
    assert rc == SD_ERR_UNSUPPORTED, msg
    with pytest.raises(capi.SdError):
        capi.final_merge(capi.product_api(), desc, b"")
    b2 = PlanBuilder()
    k, x = b2.col(T.INT, 0, True), b2.col(T.DOUBLE, 1, True)
    b2.rollup(k)
    for _ in range(17):
        b2.var_samp(x)   # one input: one shift
    assert _codegen(b2.build())[0] == 0
