"""Builds tests/golden/tpch_lineitem.npz from the reference's own TPC-H fixture.  The tests read only the
stored .npz; this script needs a SnappyData source checkout, given as its argument:

  usage   python tests/golden/make_tpch_golden.py SNAPPYDATA_CHECKOUT
  input   SNAPPYDATA_CHECKOUT/tests/common/src/main/resources/TPCH/lineitem.tbl        (30,201 rows)
  golden  SNAPPYDATA_CHECKOUT/tests/common/src/main/resources/TPCH/RESULT/Snappy_1.out, Snappy_6.out
          (the expected lines TPCHDUnitTest compares against,
           cluster/src/dunit/scala/org/apache/spark/sql/TPCHDUnitTest.scala:643-700)

The .tbl rows are encoded with snappydata_b200.column_format into real ColumnBatch bytes for the 7
columns Q1/Q6 read (5 buckets like the dunit test, batches of <= 4096 rows so several batches and
per-batch dictionaries occur); the 9 unread table columns are left empty.  The fixture stores the
encoded buffers, not the text.
"""
import datetime
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from snappydata_b200.column_format import SqlType, build_batch  # noqa: E402

TPCH = os.path.join("tests", "common", "src", "main", "resources", "TPCH")
EPOCH = datetime.date(1970, 1, 1)


def main(checkout):
    REF = os.path.join(checkout, TPCH)
    rows = [l.rstrip("\n").split("|") for l in open(os.path.join(REF, "lineitem.tbl"))]
    n = len(rows)
    orderkey = np.array([int(r[0]) for r in rows])
    data = {
        "l_quantity": np.array([float(r[4]) for r in rows]),
        "l_extendedprice": np.array([float(r[5]) for r in rows]),
        "l_discount": np.array([float(r[6]) for r in rows]),
        "l_tax": np.array([float(r[7]) for r in rows]),
        "l_returnflag": np.array([r[8].encode() for r in rows], dtype="S1"),
        "l_linestatus": np.array([r[9].encode() for r in rows], dtype="S1"),
        "l_shipdate": np.array([(datetime.date.fromisoformat(r[10]) - EPOCH).days for r in rows], dtype=np.int32),
    }
    schema = [("l_quantity", SqlType.DOUBLE, False), ("l_extendedprice", SqlType.DOUBLE, False),
              ("l_discount", SqlType.DOUBLE, False), ("l_tax", SqlType.DOUBLE, False),
              ("l_returnflag", SqlType.STRING, False), ("l_linestatus", SqlType.STRING, False),
              ("l_shipdate", SqlType.DATE, False)]
    nbuckets, per_batch = 5, 4096
    out = {}
    nb = 0
    for bucket in range(nbuckets):
        sel = np.flatnonzero(orderkey % nbuckets == bucket)          # PARTITION_BY l_orderkey
        for s in range(0, sel.shape[0], per_batch):
            idx = sel[s: s + per_batch]
            b = build_batch(idx.shape[0], schema, {k: v[idx] for k, v in data.items()}, batch_id=nb, bucket_id=bucket)
            for c, buf in enumerate(b.columns):
                out[f"b{nb}_c{c}"] = np.frombuffer(buf, dtype=np.uint8)
            out[f"b{nb}_meta"] = np.array([idx.shape[0], bucket], dtype=np.int64)
            nb += 1
    out["num_batches"] = np.array([nb])
    out["num_rows"] = np.array([n])
    out["snappy_1_out"] = np.frombuffer(open(os.path.join(REF, "RESULT/Snappy_1.out"), "rb").read(), dtype=np.uint8)
    out["snappy_6_out"] = np.frombuffer(open(os.path.join(REF, "RESULT/Snappy_6.out"), "rb").read(), dtype=np.uint8)
    dst = os.path.join(ROOT, "tests", "golden", "tpch_lineitem.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: {n} rows, {nb} batches, {os.path.getsize(dst)} bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
