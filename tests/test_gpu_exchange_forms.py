"""sd_plan_exchange on one rank: a dense / no-key plan sends its raw device state unless an aggregate holds its value as a
device record address (STRING MIN / MAX, FIRST / LAST of a STRING), which only means something on the rank that holds the
record; those plans go by value.  Either form must give the rows the plan gives without an exchange."""
import pytest

from helpers import assert_rowsets_match
from snappydata_b200 import capi, lineitem, plan as P
from snappydata_b200.column_format import SqlType as T
from snappydata_b200.plan import PlanBuilder


def _plan(keyed, ref):
    b = PlanBuilder()
    rf, ls, qty = b.col(T.STRING, P.L_RETURNFLAG), b.col(T.STRING, P.L_LINESTATUS), b.col(T.DOUBLE, P.L_QUANTITY)
    if keyed:
        b.group_by(rf)
    b.count().sum(qty).min(qty)
    if ref:
        b.max(ls).min(ls).first(ls).last(ls, ignore_nulls=True)
    return b.build(), (1 if keyed else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("keyed", [True, False], ids=["dense", "nokey"])
@pytest.mark.parametrize("ref", [True, False], ids=["record_address", "words"])
def test_single_rank_exchange_matches_the_plan_without_one(gpu_api, keyed, ref, monkeypatch):
    table = lineitem.gen_table(90_001, 20_000, seed=5)
    comm = capi.Comm(gpu_api, 0, 1, 0, lambda b: b)
    try:
        desc, nk = _plan(keyed, ref)
        plain = capi.Plan(gpu_api, desc).set_literals([])
        for b in table:
            plain.submit(b)
        want = plain.final_merge(plain.finish_raw())
        plain.close()
        assert all(v is not None for r in want for v in r), want
        for rows_form in (False, True):
            if rows_form:
                monkeypatch.setenv("SD_TUNE_EXCHANGE_ROWS", "1")
            else:
                monkeypatch.delenv("SD_TUNE_EXCHANGE_ROWS", raising=False)
            gp = capi.Plan(gpu_api, desc).set_literals([])
            for b in table:
                gp.submit(b)
            gp.exchange(comm)
            got = gp.final_merge(gp.finish_raw())
            gp.close()
            assert_rowsets_match(got, want, nk)
    finally:
        comm.close()
