"""One rank of a multi-rank test under torchrun (one process per GPU): ``python rank_worker.py <test module>`` runs
``on_ranks(pm, comm)`` of that module in tests/ on the world communicator.  Started by op_checks.run_on_ranks."""
import importlib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(HERE, "golden")]

import torch  # noqa: E402

import pylops_mpi_b200 as pm  # noqa: E402

name = sys.argv[1]
comm = pm.get_comm_world()
importlib.import_module(name).on_ranks(pm, comm)
comm.Barrier()
torch.cuda.synchronize()
print(f"RANK_WORKER_OK {name} rank={comm.Get_rank()} size={comm.Get_size()}")
