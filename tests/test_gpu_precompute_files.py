"""Analyzer.precompute_files against the precompute_file loop (the reference's `precompute`): the
same files written, byte for byte, and the same messages, for hashes at shifts 1 and 4 and for
peaks, with skip_existing over pre-existing and same-list outputs, overwrites, zero-length analyses
and a read failure; wavfiles2peaks against wavfile2peaks per file; the files, messages, tables
and match lines of the reference's own precompute -> new -> merge -> match sequence
(tests/golden/precompute.npz); and dist.precompute_files_sharded at world 1 and at world 2 over gloo."""
import contextlib
import datetime
import io
import os
import random
import shutil
import socket
import wave

import numpy as np
import pytest

from audfprint_b200 import Analyzer, HashTable
from audfprint_b200 import dist as afd
from tests.test_gpu_ingest_files import files  # noqa: F401  (the mixed list fixture)

pytestmark = pytest.mark.gpu


def _tree(root):
    out = {}
    for dp, _, fns in os.walk(root):
        for fn in fns:
            p = os.path.join(dp, fn)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def _an(shifts):
    an = Analyzer(density=100.0)
    an.shifts = shifts
    an.fail_on_error = False
    return an


def _run(lst, outdir, shifts, listed, **kw):
    an = _an(shifts)
    if listed:
        msgs = an.precompute_files(lst, str(outdir), **kw)
    else:
        msgs = [an.precompute_file(f, str(outdir), **kw) for f in lst]
    return msgs, _tree(outdir), (an.soundfiledur, an.soundfiletotaldur, an.soundfilecount)


def _strip_mixed(files):
    d, names, mixed = files
    # names repeated in the list write the same output (the later one overwrites)
    return d, [f for f in mixed if not f.endswith("rate0.wav")] + [names[2]]


@pytest.mark.parametrize("type_,shifts", [("hashes", 1), ("hashes", 4), ("peaks", 1)])
def test_precompute_files_equals_loop(files, tmp_path, type_, shifts):
    d, lst = _strip_mixed(files)
    a = _run(lst, tmp_path / "a", shifts, False, type=type_, strip_prefix=str(d))
    b = _run(lst, tmp_path / "b", shifts, True, type=type_, strip_prefix=str(d))
    assert a[0] == [[m.replace(str(tmp_path / "b"), str(tmp_path / "a")) for m in ms] for ms in b[0]]
    assert a[1] == b[1]
    assert a[2] == b[2]
    assert any(m[0].startswith("Zero length analysis") for m in b[0])


def test_skip_existing(files, tmp_path):
    d, names, _ = files
    lst = [names[0], names[1], names[0], names[2], names[1], names[3]]
    for listed, sub in ((False, "a"), (True, "b")):
        out = tmp_path / sub
        out.mkdir()
        pre = Analyzer(density=100.0).precompute_file(names[3], str(out), strip_prefix=str(d))
        assert pre[0].startswith("wrote")
    a = _run(lst, tmp_path / "a", 1, False, skip_existing=True, strip_prefix=str(d))
    b = _run(lst, tmp_path / "b", 1, True, skip_existing=True, strip_prefix=str(d))
    fix = lambda ms: [[m.replace(str(tmp_path / "b"), str(tmp_path / "a")) for m in x] for x in ms]
    assert a[0] == fix(b[0])
    assert sum("skipping" in m[0] for m in a[0]) == 3
    assert a[1] == b[1] and a[2] == b[2]


def test_read_failure(files, tmp_path):
    d, names, _ = files
    lst = [names[0], names[1], str(d / "broken.wav"), names[2]]
    errs, trees = [], []
    for listed, sub in ((False, "a"), (True, "b")):
        an = _an(1)
        an.fail_on_error = True
        out = tmp_path / sub
        with pytest.raises(IOError) as ei:
            if listed:
                an.precompute_files(lst, str(out), strip_prefix=str(d))
            else:
                for f in lst:
                    an.precompute_file(f, str(out), strip_prefix=str(d))
        errs.append(str(ei.value))
        trees.append(_tree(out))
    assert errs[0] == errs[1] and trees[0] == trees[1] and len(trees[0]) == 2


@pytest.mark.parametrize("shifts", [None, 1, 4])
def test_wavfiles2peaks_equals_per_file(files, shifts):
    d, lst = _strip_mixed(files)
    lst = [f for f in lst if not f.endswith(".afpt")]
    a, b = _an(4), _an(4)
    want = [a.wavfile2peaks(f, shifts) for f in lst]
    got = b.wavfiles2peaks(lst, shifts)
    assert got == want
    assert (a.soundfiledur, a.soundfiletotaldur, a.soundfilecount) == \
        (b.soundfiledur, b.soundfiletotaldur, b.soundfilecount)


def test_precompute_files_sharded_world1(files, tmp_path):
    d, lst = _strip_mixed(files)
    a = _run(lst, tmp_path / "a", 1, True, strip_prefix=str(d))
    msgs = afd.precompute_files_sharded(_an(1), lst, str(tmp_path / "b"), strip_prefix=str(d))
    fix = lambda ms: [[m.replace(str(tmp_path / "b"), str(tmp_path / "a")) for m in x] for x in ms]
    assert fix(msgs) == a[0]
    assert _tree(tmp_path / "b") == a[1]
    shutil.rmtree(tmp_path / "b")


# ---- the reference's own precompute -> new -> merge -> match (tests/golden/precompute.npz) -------
@pytest.fixture(scope="module")
def gp():
    from tests.conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "precompute.npz")), np.load(os.path.join(GOLDEN, "bundled.npz"))


@pytest.fixture
def refdir(gp, tmp_path, monkeypatch):
    """The fixture's WAVs (from the committed PCM), written in its relative layout; cwd inside."""
    g, gb = gp
    pcms = [gb["track%d/pcm" % k] for k in (0, 4, 8, 12)] + [gb["query/pcm"]]
    names = [str(t) for t in g["tracks"]] + [str(g["query"])]
    for nm, pcm in zip(names, pcms):
        fn = tmp_path / nm
        fn.parent.mkdir(parents=True, exist_ok=True)
        with wave.open(str(fn), "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(11025)
            w.writeframes(np.ascontiguousarray(pcm, np.int16).tobytes())
    monkeypatch.chdir(tmp_path)
    return names


RUNS = {"hashes_s1": ("hashes", 1, "precompdir"), "hashes_s4": ("hashes", 4, "precompdir_s4"),
        "peaks_s1": ("peaks", 1, "precomppkdir")}


@pytest.mark.parametrize("key", sorted(RUNS))
@pytest.mark.parametrize("listed", [False, True])
def test_precompute_equals_reference(gp, refdir, key, listed):
    g, _ = gp
    type_, shifts, pdir = RUNS[key]
    an = _an(shifts)
    with contextlib.redirect_stdout(io.StringIO()):
        if listed:
            msgs = an.precompute_files(refdir, pdir, type=type_)
        else:
            msgs = [an.precompute_file(f, pdir, type=type_) for f in refdir]
    assert [m[0] for m in msgs] == [str(m) for m in g[key + "/msgs"]]
    outs = [str(o) for o in g[key + "/outputs"]]
    assert sorted(_tree(pdir)) == sorted(os.path.relpath(o, pdir) for o in outs)
    for o in outs:
        assert open(o, "rb").read() == g["%s/%s" % (key, o)].tobytes(), o


def _write_fixture_files(g):
    for key in RUNS:
        for o in g[key + "/outputs"]:
            o = str(o)
            os.makedirs(os.path.dirname(o), exist_ok=True)
            open(o, "wb").write(g["%s/%s" % (key, o)].tobytes())


def _table_equals(ht, g, key):
    b = g[key + "/buckets"]
    counts = np.asarray(ht.counts)
    assert np.array_equal(np.nonzero(counts)[0], b)
    np.testing.assert_array_equal(np.asarray(ht.table)[b], g[key + "/rows"])
    np.testing.assert_array_equal(counts[b], g[key + "/counts"])
    assert list(ht.names) == [str(n) for n in g[key + "/names"]]
    np.testing.assert_array_equal(np.asarray(ht.hashesperid, np.uint32), g[key + "/hashesperid"])


@pytest.mark.parametrize("route", ["precomp", "precomppk"])
def test_new_merge_match_from_precomputed_files(gp, refdir, route):
    """`new` from two tracks' precomputed files, `new` from the other two, `merge`, `match` of the
    query's precomputed file: the reference's tables, "Added" lines and report lines."""
    from tests.test_gpu_zz_bundled import make_matcher
    g, _ = gp
    _write_fixture_files(g)
    ext = ".afpk" if route == "precomppk" else ".afpt"
    pdir = "precomppkdir" if route == "precomppk" else "precompdir"
    files = [os.path.join(pdir, os.path.splitext(t)[0] + ext) for t in refdir[:4]]
    random.seed(2015)
    np.random.seed(2015)
    tabs, lines = [], []
    for k, part in enumerate((files[:2], files[2:])):
        an = _an(1)
        ht = HashTable(hashbits=20, depth=100, maxtime=16384)
        tot = sum(nh for _, nh in an.ingest_files(ht, part))
        lines.append("Added " + str(tot) + " hashes " + "(%.1f" % (tot / float(an.soundfiletotaldur)) + " hashes/sec)")
        _table_equals(ht, g, "%s/new%d" % (route, k))
        tabs.append(ht)
    assert lines == [str(x) for x in g[route + "/new_lines"]]
    tabs[1].merge_batch([tabs[0]])
    _table_equals(tabs[1], g, route + "/merged")
    qan = _an(4)
    with contextlib.redirect_stdout(io.StringIO()):
        got = make_matcher().files_match_to_msgs(qan, tabs[1], [str(g[route + "/qfile"])])
    assert [m for ms in got for m in ms] == [str(x) for x in g[route + "/match_lines"]]


# ---- world 2 over gloo, spawned on one GPU -------------------------------------------------------
def _worker(rank, world, port, where, names, fail, out):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["AFP_DEVICE"] = "0"
    torch.cuda.set_device(0)
    os.chdir(where)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        an = Analyzer(density=100.0, device=0)
        an.fail_on_error = fail
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                got = afd.precompute_files_sharded(an, names, "w2", strip_prefix=None)
            out.put((rank, "ok", got))
        except Exception as e:
            out.put((rank, type(e).__name__, str(e)))
    finally:
        dist.destroy_process_group()


def _spawn(target, args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=target, args=(r, 2, port) + args + (out,)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = sorted((out.get(timeout=600) for _ in range(2)), key=lambda t: t[0])
        for p in procs:
            p.join(600)
            assert p.exitcode == 0
        return res
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)


def test_precompute_files_sharded_world2_gloo(files, tmp_path):
    d, names, _ = files
    rel = [os.path.basename(n) for n in names]
    # repeated outputs: every file of one output runs on one rank, in list order
    lst = rel + [rel[1], "empty.wav", rel[4], "broken.wav", rel[0]]
    cwd = os.getcwd()
    os.chdir(d)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            want = _an(1).precompute_files(lst, str(tmp_path / "one"))
        want_tree = _tree(str(tmp_path / "one"))
    finally:
        os.chdir(cwd)
    shutil.rmtree(d / "w2", ignore_errors=True)
    res = _spawn(_worker, (str(d), lst, False))
    assert res[0][1] == "ok" and res[1][1] == "ok" and res[1][2] is None
    fix = lambda ms: [[m.replace("w2/", str(tmp_path / "one") + "/") for m in x] for x in ms]
    assert fix(res[0][2]) == want
    assert _tree(str(d / "w2")) == want_tree
    shutil.rmtree(d / "w2")
    res = _spawn(_worker, (str(d), rel[:3] + ["broken.wav"] + rel[3:], True))      # index 3: rank 1's file
    assert [r[1] for r in res] == ["OSError", "OSError"]
    assert res[0][2] == res[1][2] == "wavfile2peaks: Error reading broken.wav"
    shutil.rmtree(d / "w2", ignore_errors=True)
