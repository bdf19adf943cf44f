"""Host-only checks of UPDATE / DELETE plans (SD_PLAN_MUTATE): the builder and the descriptor, and an NVRTC compile for sm_90a of
the generated source of mutation plans in all four kernel variants (SET targets of every fixed-width type, nullable and not, and
a DELETE)."""
import pytest

from snappydata_b200 import capi
from snappydata_b200.column_format import SqlType as T
from snappydata_b200.plan import PlanBuilder

FIXED = [T.BYTE, T.SHORT, T.INT, T.LONG, T.FLOAT, T.DOUBLE, T.DATE, T.TIMESTAMP, T.DECIMAL]


def _update_every_type():
    # every fixed-width type twice: table column 2k NOT NULL, 2k + 1 nullable
    b = PlanBuilder()
    types = [t for t in FIXED for _ in (0, 1)]
    cols = [b.col(t, i, i % 2 == 1, scale=2 if t == T.DECIMAL else 0, precision=12 if t == T.DECIMAL else 0) for i, t in enumerate(types)]
    b.filter(cols[4] > b.lit(T.INT))
    b.update({i: (c + c if t not in (T.DATE, T.TIMESTAMP, T.DECIMAL) else c) for i, (c, t) in enumerate(zip(cols, types))})
    return b.build()


def _delete():
    b = PlanBuilder()
    d = b.col(T.DATE, 10)
    b.filter(d < b.lit(T.DATE))
    b.delete()
    return b.build()


def test_builder_sets_the_flag_and_targets():
    d = _update_every_type()
    assert d.c.flags == capi.SD_PLAN_MUTATE and d.flags == capi.SD_PLAN_MUTATE
    assert d.targets == list(range(2 * len(FIXED))) and d.c.nproj == 2 * len(FIXED)
    assert [c[1] for c in d.cols_py] == [i % 2 == 1 for i in range(2 * len(FIXED))]
    x = _delete()
    assert x.c.flags == capi.SD_PLAN_MUTATE and x.c.nproj == 0 and x.targets == [] and x.c.naggs == 0 and x.c.nkeys == 0
    b = PlanBuilder()
    b.count(b.col(T.INT, 0))
    assert b.build().c.flags == 0


@pytest.mark.parametrize("label", ["update", "delete"])
def test_mutation_kernels_compile_for_sm_90a(label):
    pytest.importorskip("cuda.bindings.nvrtc")
    from test_jit_compiles import _codegen, _compile   # the NVRTC harness of the plan compile test
    desc = _update_every_type() if label == "update" else _delete()
    seen = set()
    for slow, litnull in ((0, 0), (1, 0), (0, 1), (1, 1)):
        source, sig, name = _codegen(desc, slow, litnull)
        assert "sd::MODE_MUTATE" in source and ";mode=4;" in sig
        assert name not in seen
        seen.add(name)
        _compile(source, name)
