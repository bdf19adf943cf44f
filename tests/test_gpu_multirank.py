"""N > 1 on hardware: the NCCL exchange behind the C ABI (sd_comm_* / sd_plan_exchange) under the driver's own launch
(torchrun, one rank per GPU).  Needs >= 2 GPUs: skipped on a single-GPU machine (bench.py's parity_check covers N > 1
whenever the bench itself is run on several GPUs)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def test_exchange_on_two_gpus_equals_the_oracle_over_the_whole_table():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29533", os.path.join(HERE, "multirank_worker.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "MULTIRANK OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
