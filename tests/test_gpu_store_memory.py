"""The resident store's device memory: slabs allocated as compressible where the device supports generic memory
compression, the bytes read back unchanged, and every slab returned when the store is destroyed."""
import ctypes as C

import pytest
import torch

from snappydata_b200 import capi, lineitem
from snappydata_b200 import plan as P

pytestmark = pytest.mark.gpu

CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED = 107


def compression_supported(device=0):
    cuda = C.CDLL("libcuda.so.1")
    dev, val = C.c_int(), C.c_int()
    assert cuda.cuInit(0) == 0
    assert cuda.cuDeviceGet(C.byref(dev), device) == 0
    assert cuda.cuDeviceGetAttribute(C.byref(val), CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, dev) == 0
    return bool(val.value)


def test_generated_store_is_compressible_and_bytes_unchanged(gpu_api):
    rows, per_batch = 600_000, 200_000
    store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    try:
        store.gen_lineitem(0, rows, per_batch, 8, 42, lineitem.Q1_COLUMN_MASK)
        comp, total = store.memory_info()
        assert total >= store.nbytes() > 0
        if compression_supported():
            assert comp == total
        else:
            assert comp == 0
        want = lineitem.gen_table(rows, per_batch, 42)
        for i, hb in enumerate(want):
            for c in (P.L_QUANTITY, P.L_EXTENDEDPRICE, P.L_DISCOUNT, P.L_TAX, P.L_RETURNFLAG, P.L_LINESTATUS, P.L_SHIPDATE):
                assert store.get_buffer(i, c) == hb.columns[c], f"batch {i} column {c}"
    finally:
        store.close()


def test_store_destroy_returns_every_slab(gpu_api):
    """A slab that holds one oversize buffer (a 70M-row l_quantity column, 560 MB) and a default-size slab after it, created
    and destroyed 20 times: free device memory comes back to where it started."""
    big = 70_000_000

    def cycle():
        store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
        try:
            store.gen_lineitem(0, big, big, 1, 3, 1 << P.L_QUANTITY)
            store.gen_lineitem(big, 400_000, 200_000, 1, 3, lineitem.Q1_COLUMN_MASK)
            comp, total = store.memory_info()
            assert total >= big * 8 + (512 << 20)
            assert comp in (0, total)
        finally:
            store.close()

    cycle()   # the first store's driver and runtime set-up is not a slab
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    for _ in range(20):
        cycle()
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    # one leaked slab per cycle would be over 20 GB; the slack is for other work on the device
    assert free0 - free1 < (256 << 20), (free0, free1)
