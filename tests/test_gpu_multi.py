"""Multi-rank parity: launches tests/multi_worker.py under torchrun with one rank per GPU.  World size 1 runs
on any GPU box (the whole worker through the torchrun/NCCL-less path); 2 / 4 / 8 need that many GPUs
(4 also covers the square-grid MPIMatrixMult paths) and are skipped otherwise."""
import os

import pytest

from op_checks import HERE, needs_gpus, run_on_ranks

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nproc", [1, 2, 4, 8])
def test_multi_rank_parity(nproc):
    needs_gpus(nproc)
    assert run_on_ranks(os.path.join(HERE, "multi_worker.py"), nproc, timeout=1500).count("MULTI_WORKER_OK") == nproc
