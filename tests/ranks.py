"""Two-rank (or `world`-rank) gloo runs on the CPU for the data-parallel tests (not collected: the name does not match
test_*.py).  A test hands `run_ranks` a module-level worker(rank, world, ret); each rank runs it in a spawned process with
the process group set up, and whatever the workers store in `ret` comes back to the test."""
import os
import socket
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT


def _free_port():
    """A port no other process holds now: one the kernel hands out for ("127.0.0.1", 0).  Fixed or pid-derived ports
    collide when two runs of the suite share a machine."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(worker, rank, world, port, ret):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    from gangealing_b200.training import distributed as gdist
    assert gdist.setup_distributed("gloo")
    worker(rank, world, ret)
    gdist.synchronize()
    dist.destroy_process_group()


def run_ranks(worker, timeout, world=2):
    """Run worker(rank, world, ret) on `world` spawned gloo ranks, join each within `timeout` seconds, assert that every
    rank exited cleanly and return a plain dict copy of `ret`."""
    ctx = mp.get_context("spawn")
    with ctx.Manager() as mgr:
        ret = mgr.dict()
        port = _free_port()
        procs = [ctx.Process(target=_rank_main, args=(worker, r, world, port, ret)) for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        return dict(ret)
