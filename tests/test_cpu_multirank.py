"""multirank.run_ranks on the CPU: every rank's outputs come back, a rank that raises fails the call at once with its own exception, a
hung rank fails it at the deadline, and no child process outlives a failed call. The workers import neither the engine nor CUDA."""
import multiprocessing
import os
import time

import pytest
import torch.multiprocessing as mp

from multirank import run_ranks

HANG = 300.0          # far past every deadline below: a rank that sleeps this long is only ever ended by run_ranks


def _echo(rank, world, rendezvous, out, tag):
    out[rank] = (world, rendezvous, tag)


def _fail_or_hang(rank, world, rendezvous, out, failing_rank):
    if rank == failing_rank:
        raise ValueError(f"rank {rank} failed on purpose")
    time.sleep(HANG)


@pytest.fixture
def child_pids(monkeypatch):
    """the pids of every rank process run_ranks starts, whether or not it reached the worker"""
    pids, start = [], multiprocessing.context.SpawnProcess.start

    def recording(self):
        start(self)
        pids.append(self.pid)
    monkeypatch.setattr(multiprocessing.context.SpawnProcess, "start", recording)
    yield pids
    assert pids and multiprocessing.active_children() == []
    for pid in pids:
        with pytest.raises(ProcessLookupError):
            os.kill(pid, 0)


def test_every_rank_returns_its_outputs():
    assert run_ranks(_echo, 3, ("x",), comm=None) == {r: (3, None, "x") for r in range(3)}


def test_a_raising_rank_fails_the_call_promptly(child_pids):
    t0 = time.monotonic()
    with pytest.raises(mp.ProcessRaisedException, match="ValueError: rank 1 failed on purpose") as exc:
        run_ranks(_fail_or_hang, 3, (1,), comm=None, timeout=HANG)
    assert exc.value.error_index == 1
    assert time.monotonic() - t0 < 60.0


def test_a_hung_rank_fails_the_call_at_the_deadline(child_pids):
    """the deadline counts from the start, so a child may still be importing torch when it is terminated: either way it is gone"""
    t0 = time.monotonic()
    with pytest.raises(TimeoutError, match="2 ranks did not finish within 5 s"):
        run_ranks(_fail_or_hang, 2, (None,), comm=None, timeout=5.0)
    assert time.monotonic() - t0 < 5.0 + 10.0
