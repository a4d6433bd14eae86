"""Host pieces of the precompute list forms: output naming (audfprint.py:76-93), the round planning
that keeps the per-file loop's skip / overwrite order effects, output ownership across ranks, and
list-order reassembly of precompute_files_sharded over gloo."""
import os
import socket

import numpy as np
import pytest
import torch.multiprocessing as mp

from audfprint_b200 import analyzer as an_mod
from audfprint_b200 import dist as afd


@pytest.mark.parametrize("fn,prefix,want", [
    ("a/b/c.wav", None, "out/a/b/c.afpt"),
    ("./a/./c.mp3", None, "out/a/c.afpt"),
    ("../../x/y.wav", None, "out/x/y.afpt"),
    ("/abs/path/t.wav", None, "out/abs/path/t.afpt"),
    ("/data/wavs/s/t.wav", "/data/wavs", "out/s/t.afpt"),
    ("/data/wavs/s/t.wav", "/data/wavs/", "out/s/t.afpt"),
    ("/data/other/t.wav", "/data/wavs", "out/data/other/t.afpt"),
    ("noext", None, "out/noext.afpt"),
    ("a.b/c.d.wav", None, "out/a.b/c.d.afpt"),
])
def test_precompute_name(fn, prefix, want):
    assert an_mod.precompute_name(fn, "out", True, prefix) == want
    assert an_mod.precompute_name(fn, "out", False, prefix) == want[:-5] + ".afpk"


def test_precompute_name_empty_dir():
    assert an_mod.precompute_name("./x/y.wav", "", True) == "x/y.afpt"


def test_round_planning_skip_and_overwrite():
    names = ["a", "b", "a", "c", "b", "d", "e"]
    on_disk = {"c"}
    # without skip_existing a repeated name stays in the round (the later file overwrites)
    assert an_mod.next_precompute_round(names, 0, False, on_disk.__contains__, 100) == (7, [])
    # with skip_existing a repeated name closes the round before it; existing outputs are skipped
    assert an_mod.next_precompute_round(names, 0, True, on_disk.__contains__, 100) == (2, [])
    # (the earlier "b" wrote in the first round, so the disk now has it)
    on_disk |= {"a", "b"}
    assert an_mod.next_precompute_round(names, 2, True, on_disk.__contains__, 100) == (7, [2, 3, 4])
    assert an_mod.next_precompute_round(names, 0, False, on_disk.__contains__, 3) == (3, [])


@pytest.mark.parametrize("world", [2, 3])
def test_owners(world):
    names = ["a", "b", "a", "c", "b", "d", "a", "e", "c"]
    owners = afd.precompute_owners(names, world)
    first = {}
    for j, n in enumerate(names):
        first.setdefault(n, j)
        assert owners[j] == first[n] % world
    # every file writing one output runs on one rank
    for n in set(names):
        assert len({int(owners[j]) for j in range(len(names)) if names[j] == n}) == 1


def _worker(rank, world, port, outdir, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        class Stub:
            """precompute_files without a device: one message per file naming it and the rank."""
            def precompute_files(self, filenames, precompdir, type, skip_existing, strip_prefix):
                return [["%s by %d" % (f, rank)] for f in filenames]
        names = ["f%d.wav" % (j % 7) for j in range(17)]
        out = afd.precompute_files_sharded(Stub(), names, outdir)
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_list_order_over_gloo(world, tmp_path):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path), q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(60)
    names = ["f%d.wav" % (j % 7) for j in range(17)]
    owners = afd.precompute_owners([an_mod.precompute_name(f, str(tmp_path)) for f in names], world)
    assert res[0] == [["%s by %d" % (f, owners[j])] for j, f in enumerate(names)]
    assert all(res[r] is None for r in range(1, world))


def test_precompute_write_bytes(tmp_path):
    """The writer emits the magic, then the int32 pairs (what hashes_save / peaks_save write)."""
    rows = np.array([[0, 5], [3, 123456], [2 ** 20, 7]], np.int32)
    a, b = str(tmp_path / "x" / "a.afpt"), str(tmp_path / "b.afpt")
    msg = an_mod._precompute_write("in.wav", a, True, rows, 1.5)
    an_mod.hashes_save(b, [tuple(r) for r in rows.tolist()])
    assert open(a, "rb").read() == open(b, "rb").read()
    assert msg == "wrote " + a + " ( 3 hashes, 1.500 sec)"
    pk = str(tmp_path / "p.afpk")
    assert an_mod._precompute_write("in.wav", pk, False, [(1, 2)], 0.25) == "wrote " + pk + " ( 1 peaks, 0.250 sec)"
    assert open(pk, "rb").read() == an_mod.PEAK_MAGIC + np.array([1, 2], "<i4").tobytes()
    assert an_mod._precompute_write("in.wav", str(tmp_path / "z.afpt"), True, [], 0.0) == \
        "Zero length analysis for in.wav -- not saving."
    assert not os.path.exists(str(tmp_path / "z.afpt"))


# ---- against the reference's own precompute (tests/golden/precompute.npz) -----------------------
@pytest.fixture(scope="module")
def gp():
    from tests.conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "precompute.npz")), np.load(os.path.join(GOLDEN, "bundled.npz"))


@pytest.mark.parametrize("key", ["hashes_s1", "hashes_s4", "peaks_s1"])
def test_host_statement_against_reference(gp, key, tmp_path):
    """Output names, file bytes and messages of the reference's precompute follow from the rows it
    computed and the file's duration: what precompute_name and the writer state."""
    g, gb = gp
    hashes = key.startswith("hashes")
    pdir = {"hashes_s1": "precompdir", "hashes_s4": "precompdir_s4", "peaks_s1": "precomppkdir"}[key]
    wavs = [str(t) for t in g["tracks"]] + [str(g["query"])]
    pcms = [gb["track%d/pcm" % k] for k in (0, 4, 8, 12)] + [gb["query/pcm"]]
    for fn, pcm, op, msg in zip(wavs, pcms, g[key + "/outputs"], g[key + "/msgs"]):
        op = str(op)
        assert an_mod.precompute_name(fn, pdir, hashes) == op
        want = g["%s/%s" % (key, op)].tobytes()
        assert want[:16] == (an_mod.HASH_MAGIC if hashes else an_mod.PEAK_MAGIC)
        rows = np.frombuffer(want[16:], "<i4").reshape(-1, 2)
        mine = str(tmp_path / op)
        got_msg = an_mod._precompute_write(fn, mine, hashes, rows, len(pcm) / 11025)
        assert got_msg == str(msg).replace(op, mine)
        assert open(mine, "rb").read() == want
        loaded = (an_mod.hashes_load if hashes else an_mod.peaks_load)(mine)
        assert loaded == [tuple(r) for r in rows.tolist()]
