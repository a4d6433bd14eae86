"""CPU: the status exchange the multi-GPU entry points (ingest_sharded, match_files_sharded,
precompute_files_sharded) end their per-rank work with - every rank raises the same thing when one
rank failed, and no rank is left inside a collective - over gloo at world size 2."""
import os
import socket

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from audfprint_b200 import dist as afd

# case -> (exception of rank 0, exception of rank 1, io_errors_everywhere)
CASES = {
    "ok": (None, None, True),
    "ioerror_everywhere": (None, IOError("wavfile2peaks: Error reading b.wav"), True),
    "ioerror_local": (None, IOError("wavfile2peaks: Error reading b.wav"), False),
    "other": (None, ValueError("signal must be 1-D"), True),
    "both": (IOError("wavfile2peaks: Error reading a.wav"), ValueError("signal must be 1-D"), True),
}


def _outcome(err, io_errors_everywhere):
    codes = afd.gather_objects(afd._status_code(err, io_errors_everywhere))
    try:
        afd._raise_if_failed(err, codes, "entry_point")
    except Exception as e:      # noqa: BLE001 - the point is to compare what is raised
        return type(e).__name__, str(e), e is err
    return None


def _worker(rank, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        got = {case: _outcome(errs[rank], errs[2]) for case, errs in CASES.items()}
        got["after"] = afd.gather_objects(rank)          # every rank left the exchanges above
        out.put((rank, got))
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module")
def outcomes():
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(out.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    assert got[0]["after"] == got[1]["after"] == [0, 1]
    return got


def test_no_failure_raises_nothing(outcomes):
    assert outcomes[0]["ok"] is None and outcomes[1]["ok"] is None


def test_ioerror_is_raised_on_every_rank(outcomes):
    msg = "wavfile2peaks: Error reading b.wav"
    assert outcomes[1]["ioerror_everywhere"] == ("OSError", msg, True)         # its own exception
    assert outcomes[0]["ioerror_everywhere"] == ("OSError", msg, False)


def test_ioerror_without_io_errors_everywhere_names_the_rank(outcomes):
    msg = "wavfile2peaks: Error reading b.wav"
    assert outcomes[1]["ioerror_local"] == ("OSError", msg, True)
    assert outcomes[0]["ioerror_local"] == ("RuntimeError", "entry_point: rank 1 failed: " + msg, False)


def test_other_failure_names_the_rank(outcomes):
    assert outcomes[1]["other"] == ("ValueError", "signal must be 1-D", True)
    assert outcomes[0]["other"] == ("RuntimeError", "entry_point: rank 1 failed: signal must be 1-D", False)


def test_failing_ranks_raise_their_own(outcomes):
    assert outcomes[0]["both"] == ("OSError", "wavfile2peaks: Error reading a.wav", True)
    assert outcomes[1]["both"] == ("ValueError", "signal must be 1-D", True)


def test_single_process():
    assert _outcome(None, True) is None
    err = ValueError("x")
    assert _outcome(err, True) == ("ValueError", "x", True)
