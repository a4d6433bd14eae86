"""CPU: the reference arm of bench.py (`--impl reference`: the reference's CPU path - the unmodified
reference when a checkout is reachable, else the oracle port - timed on the host cores) prints ONE
JSON line with the keys a caller of the benchmark reads."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--files", "8",
                          "--seconds", "6", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "audio_seconds_fingerprinted_per_sec"
    assert d["unit"] == "audio-s/s" and d["higher_is_better"] is True and d["n_gpus"] == 1
    assert d["steps"] == 1 and d["warmup"] == 1 and d["value"] > 0 and d["ms_per_step"] > 0
    # the unmodified reference where $AFP_REFERENCE names a checkout, the oracle port otherwise
    ref = os.environ.get("AFP_REFERENCE")
    want_kind = "reference" if ref and os.path.isfile(os.path.join(ref, "audfprint_analyze.py")) else "port"
    assert d["cpu_baseline"]["kind"] == want_kind and d["cpu_baseline"]["cores"] >= 1
    assert d["cpu_baseline"]["host_cores"]["used"] == d["cpu_baseline"]["cores"]
    assert d["config0"]["cores"] == 1 and d["config0"]["median_s"] > 0 and d["config0"]["runs"] >= 5
    assert d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and d["vs_baseline"] is None


def test_dump_outputs_writes_float64_files_within_the_size_cap(tmp_path, monkeypatch):
    """bench.py --dump-outputs: every file when they fit, else the same seeded sample of whole
    files on every run, never more than DUMP_BYTES."""
    sys.path.insert(0, ROOT)
    import bench
    rng = np.random.default_rng(3)
    counts = rng.integers(0, 40, 50)
    roff = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    rows = rng.integers(0, 1 << 20, (int(roff[-1]), 2)).astype(np.int32)
    bench.dump_outputs(str(tmp_path / "all"), rows, roff)
    got = {n: np.load(tmp_path / "all" / (n + ".npy")) for n in ("hashes", "row_offsets", "files")}
    assert all(v.dtype == np.float64 for v in got.values())
    assert np.array_equal(got["hashes"], rows) and np.array_equal(got["row_offsets"], roff)
    assert np.array_equal(got["files"], np.arange(50))
    monkeypatch.setattr(bench, "DUMP_BYTES", 4096)
    for d in ("s1", "s2"):
        bench.dump_outputs(str(tmp_path / d), rows, roff)
    files = [np.load(tmp_path / d / "files.npy") for d in ("s1", "s2")]
    assert np.array_equal(files[0], files[1]) and 0 < len(files[0]) < 50
    h, o = np.load(tmp_path / "s1" / "hashes.npy"), np.load(tmp_path / "s1" / "row_offsets.npy")
    assert sum(os.path.getsize(tmp_path / "s1" / (n + ".npy")) - 128 for n in ("hashes", "row_offsets", "files")) <= 4096
    for k, i in enumerate(files[0].astype(int)):
        assert np.array_equal(h[int(o[k]):int(o[k + 1])], rows[roff[i]:roff[i + 1]])
