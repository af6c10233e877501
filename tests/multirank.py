"""One process per rank for the multi-rank tests, with a deadline.

run_ranks starts `world` spawned processes, each calling worker(rank, world, rendezvous, out, *args), where `out` is a manager dict the
ranks write their results into. A rank that raises fails the call with torch's ProcessRaisedException (that rank's traceback), and the
other ranks are terminated. Ranks that are all alive but never finish (a collective some rank never entered) fail the call with
TimeoutError once the deadline passes. Every child is gone when run_ranks returns or raises."""
import ctypes
import tempfile
import time

import pytest
import torch
import torch.multiprocessing as mp


def run_ranks(worker, world, args=(), *, comm, timeout=900.0):
    """dict(out) of one run of `world` ranks; `comm` chooses the rendezvous each rank gets:
      "nccl": an NCCL unique id (None at world == 1); skips the test when fewer than `world` GPUs are present,
      "gloo": a file:// init method for torch.distributed in a temporary directory,
      None:   None."""
    if comm == "nccl" and torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    with tempfile.TemporaryDirectory(prefix="multirank-") as tmp:
        rendezvous = None
        if comm == "nccl" and world > 1:
            from hiop_b200 import _lib
            buf = ctypes.create_string_buffer(128)
            _lib.check(_lib.lib().hb_comm_unique_id(buf), "hb_comm_unique_id")
            rendezvous = buf.raw
        elif comm == "gloo":
            rendezvous = f"file://{tmp}/rendezvous"
        with mp.Manager() as mgr:
            out = mgr.dict()
            pc = mp.start_processes(worker, args=(world, rendezvous, out, *args), nprocs=world, join=False, start_method="spawn")
            deadline = time.monotonic() + timeout
            try:
                while not pc.join(timeout=max(1.0, deadline - time.monotonic())):
                    if time.monotonic() >= deadline:
                        raise TimeoutError(f"the {world} ranks did not finish within {timeout:g} s (a collective that never completed?)")
            finally:
                for p in pc.processes:
                    if p.is_alive():
                        p.terminate()
                for p in pc.processes:
                    p.join(30)
                    if p.is_alive():                # stuck in native code that does not return to the SIGTERM handler
                        p.kill()
                        p.join()
            return dict(out)
