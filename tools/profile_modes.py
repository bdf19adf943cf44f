"""One launch of every kernel mode that bench.py's headline does not show, for `ncu --set full`:
  MODE_PROJECT + NULL-aware staged path (C4 wide table), staged ring + delta/delete overlay (C5 hybrid Q6), MODE_HASH
  (group by l_shipdate: ~2500 groups), the LZ4 expansion kernel (dense shape + window parse) on stored Q1 buffers.
usage: ncu --set full --clock-control none --import-source on -k regex:"scan_aggregate|lz4_decode" -o modes python tools/profile_modes.py"""
import copy
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from snappydata_b200 import capi, lineitem, plan as P, workloads as W  # noqa: E402
from snappydata_b200.column_format import SqlType as T, compress_lz4  # noqa: E402
from snappydata_b200.plan import PlanBuilder  # noqa: E402

api = capi.product_api()
api.check(api.init(0))
NB = int(sys.argv[1]) if len(sys.argv) > 1 else 24

# ---- C4: projection over a wide table, nullable columns -------------------------------------------------------------
store = capi.Store(api, [(W.C4_TYPES[i], i % 4 == 0) for i in range(128)], 0)
for k in range(NB):
    cb, _ = W.c4_base_batch(k % 6)
    cb = copy.copy(cb); cb.batch_id = k
    store.put(cb)
gp = capi.Plan(api, W.c4_plan())
gp.reset().set_literals(W.C4_LITS); gp.scan_store(store); gp.finish_raw()
m = gp.metrics()
print("c4 project", gp.kernel_name(), m["aggTimeNs"] / 1e6, "ms", m["algorithmicBytes"] / max(1, m["aggTimeNs"]), "GB/s", m["numOutputRows"], "rows out")
store.close()

# ---- C5: Q6 with deltas + deletes (overlay path) ---------------------------------------------------------------------
r = np.random.default_rng(5)
hy = [W._decorate_hybrid(b, r) for b in lineitem.gen_table(NB * 200_000, 200_000, seed=6, column_mask=lineitem.Q6_COLUMN_MASK)]
store = capi.Store(api, lineitem.LINEITEM_SCHEMA, 0)
for b in hy:
    store.put(b)
gp = capi.Plan(api, P.q6_plan())
gp.reset().set_literals(P.Q6_LITERALS); gp.scan_store(store); gp.finish_raw()
m = gp.metrics()
print("c5 overlay", gp.kernel_name(), m["aggTimeNs"] / 1e6, "ms", m["algorithmicBytes"] / max(1, m["aggTimeNs"]), "GB/s")
store.close()

# ---- MODE_HASH: group by l_shipdate ----------------------------------------------------------------------------------
store = capi.Store(api, lineitem.LINEITEM_SCHEMA, 0)
store.gen_lineitem(0, NB * 200_000, 200_000, 8, 1, lineitem.Q1_COLUMN_MASK)
b = PlanBuilder()
ship, qty, price = b.col(T.DATE, P.L_SHIPDATE), b.col(T.DOUBLE, P.L_QUANTITY), b.col(T.DOUBLE, P.L_EXTENDEDPRICE)
b.group_by(ship); b.count().sum(qty).sum(price)
gp = capi.Plan(api, b.build())
gp.reset().set_literals([]); gp.scan_store(store); raw = gp.finish_raw()
m = gp.metrics()
print("hash group-by", gp.kernel_name(), m["aggTimeNs"] / 1e6, "ms", m["algorithmicBytes"] / max(1, m["aggTimeNs"]), "GB/s", m["numOutputRows"], "groups")

# ---- LZ4: stored Q1 buffers expanded on the device -----------------------------------------------------------------------
cols = P.q1_plan().table_cols
gp = capi.Plan(api, P.q1_plan())
gp.set_option(capi.SD_OPT_RETAIN_BUFFERS, 1)
keep = []
gp.reset().set_literals(P.Q1_LITERALS)
from snappydata_b200.column_format import ColumnBatch  # noqa: E402
for i in range(store.num_batches()):
    n, bucket, bid = store.batch_info(i)
    bufs = [None] * 16
    for c in cols:
        bufs[c] = compress_lz4(store.get_buffer(i, c))
    cb = ColumnBatch(num_rows=n, columns=bufs, batch_id=bid, bucket_id=bucket)
    mb = capi.MarshalledBatch(cb, cols)
    keep.append(mb)
    gp.submit_marshalled(mb)
gp.finish_raw()
print("lz4 e2e launches", gp.metrics()["kernelLaunches"])
