"""Worker of tests/test_gpu_covariance.py (launched under torchrun, one rank per GPU): every rank scans half of the batches, and
sd_plan_exchange merges the covariance buffers of both ranks -- each rank's shifted sums converted with its own Kx / Ky -- in the
dense form (dictionaries + raw device state) and by value.  The merged result must equal one GPU's result over all the batches."""
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from snappydata_b200 import capi  # noqa: E402
from test_gpu_covariance import cov_plan, numeric_batch  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
api = capi.product_api()
api.check(api.init(local))


def bcast(b):
    box = [b]
    dist.broadcast_object_list(box, src=0)
    return box[0]


def same(x, y):
    """two results of one group: equal to the bar of the merge (1e-9 relative, or both NULL / NaN)"""
    if x is None or y is None:
        return x is None and y is None
    if math.isnan(x) or math.isnan(y):
        return math.isnan(x) and math.isnan(y)
    return abs(x - y) <= 1e-9 * max(abs(x), abs(y), 1e-300) or abs(x - y) <= 1e-12


comm = capi.Comm(api, rank, world, local, bcast)
batches = [numeric_batch(40000, "fast_nulls", seed=70 + i, groups=12, profile=("big_mean_09", "mixed")[i % 2], batch_id=i)[0]
           for i in range(6)]
mine = batches[rank::world]
for keys in ([], ["k"]):
    desc = cov_plan(keys)
    one = capi.Plan(api, desc)
    for b in batches:
        one.submit(b)
    want = sorted(one.final_merge(one.finish_raw()), key=repr)
    one.close()
    for form in ("dense", "rows"):
        if form == "rows":
            os.environ["SD_TUNE_EXCHANGE_ROWS"] = "1"
        else:
            os.environ.pop("SD_TUNE_EXCHANGE_ROWS", None)
        gp = capi.Plan(api, desc)
        for b in mine:
            gp.submit(b)
        gp.exchange(comm)
        got = sorted(gp.final_merge(gp.finish_raw()), key=repr)
        gp.close()
        nk = len(keys)
        assert [r[:nk + 1] for r in got] == [r[:nk + 1] for r in want], (keys, form)
        for a, b in zip(got, want):
            for x, y in zip(a[nk + 2:], b[nk + 2:]):   # STDDEV, COVAR_POP, COVAR_SAMP, CORR (SUM's order differs)
                assert same(x, y), (keys, form, a[:nk], x, y)
        if rank == 0:
            print(keys, form, "ok:", len(got), "groups", flush=True)
os.environ.pop("SD_TUNE_EXCHANGE_ROWS", None)
dist.barrier()
dist.destroy_process_group()
if rank == 0:
    print("COVARIANCE MULTIRANK OK", flush=True)
