"""CPU: `--king-table-require` / `--king-table-require-xor` through the host program, replayed without a GPU.  The
test-only stand-in library (tests/harness/mock_pl2gpu.cc, plain-loop KING counts, extended by
tests/harness/mock_king_mapped.cc with the mapped job over a device sample order) is injected with LD_PRELOAD, so the real driver runs: ID loading, the choice between the pair
list (a subset file or rel-check) and the mapped dense job, pass planning, the mapping of device positions back to
samples, the orientation of every pair and the sort into the reference's natural-order rows.  Every table must be
byte-identical to the one the reference binary wrote (tests/golden/make_king_require_set.py), which pins the pair
order and orientation.  The flag checks and refusals are checked for exit code and message."""
import gzip
import hashlib
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
GOLD = json.load(open(os.path.join(GD, "kr_digests.json")))
DENSE = {name for name, args in GOLD["runs"].items() if "--king-table-subset" not in args and "rel-check" not in args}


@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mock") / "mock_king_mapped.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", "mock_king_mapped.cc")], check=True)
    return so


def _run(mock_so, args, out, log=None, devices=1, mem_mib=None):
    env = dict(os.environ, LD_PRELOAD=mock_so, PL2_MOCK_DEVICES=str(devices))
    if log:
        env["PL2_MOCK_LOG"] = log
    if mem_mib:
        env["PL2_MOCK_MEM_MIB"] = str(mem_mib)
    return subprocess.run([BIN] + args + ["--out", out], capture_output=True, text=True, env=env, cwd=GD)


def _digest(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


@pytest.mark.parametrize("name", sorted(GOLD["runs"]))
def test_replay_matches_reference(mock_so, tmp_path, name):
    out, log = str(tmp_path / "o"), str(tmp_path / "mock.log")
    r = _run(mock_so, GOLD["runs"][name], out, log=log)
    assert r.returncode == 0, r.stdout + r.stderr
    assert _digest(out + ".kin0") == GOLD["digests"][name]["sha256"]
    small = os.path.join(GD, name + ".kin0.gz")
    if os.path.exists(small):
        assert open(out + ".kin0", "rb").read() == gzip.open(small).read()
    calls = [ln.split()[0] for ln in open(log)]
    if name in DENSE:
        # required pairs never become a pair list without a subset file or rel-check
        assert "king_begin_mapped" in calls and "king_pairs_begin" not in calls
    else:
        assert "king_pairs_begin" in calls and "king_begin_mapped" not in calls


def test_loaded_count_logged(mock_so, tmp_path):
    r = _run(mock_so, GOLD["runs"]["kr_req2"], str(tmp_path / "o"))
    n_req = sum(1 for ln in open(os.path.join(GD, "kr_req.txt")) if not ln.startswith("#"))
    assert "--king-table-require: %d sample IDs loaded." % n_req in r.stdout
    r = _run(mock_so, GOLD["runs"]["kr_one"], str(tmp_path / "o"))
    assert "--king-table-require: 1 sample ID loaded." in r.stdout


@pytest.mark.parametrize("name", ["kr_req", "kr_xor"])
def test_multipass_matches_reference(mock_so, tmp_path, name):
    """A device budget too small for the whole slab: the rows are split into passes, each re-streaming the variants."""
    out, log = str(tmp_path / "o"), str(tmp_path / "mock.log")
    r = _run(mock_so, GOLD["runs"][name], out, log=log, mem_mib=12)
    assert r.returncode == 0, r.stdout + r.stderr
    passes = sum(1 for ln in open(log) if ln.startswith("king_begin_mapped"))
    assert passes >= 2 and ("%d passes over the variants" % passes) in r.stdout
    assert _digest(out + ".kin0") == GOLD["digests"][name]["sha256"]


REQ = ["--bfile", "kr", "--make-king-table"]


@pytest.mark.parametrize(
    "args,code,msg",
    [
        (REQ + ["--king-table-require", "kr_req.txt", "--king-table-require-xor", "kr_req.txt"], 8, "Error: --king-table-require cannot be used with --king-table-require-xor."),
        (REQ + ["--king-table-require", "kr_req.txt", "--king-cutoff", "0.1"], 8, "Error: --king-table-require[-xor] cannot be used with --king-cutoff."),
        (REQ + ["--king-table-require-xor", "kr_req.txt", "--make-king"], 8, "Error: --make-king cannot be used with --king-table-subset or\n--king-table-require[-xor]."),
        (["--bfile", "kr", "--make-king-table", "cols=nsnp,kinship", "--king-table-require", "kr_req.txt"], 8, "Error: --king-table-require[-xor] requires --make-king-table cols= to include\nthe 'id' column set."),
        (REQ + ["--king-table-require"], 8, "--king-table-require requires at least one filename."),
        (REQ + ["--king-table-require", "kr_req.txt", "--parallel", "1", "2"], 63, "Error: --king-table-require[-xor] with --parallel is not supported by plink2_b200 yet."),
        (REQ + ["--king-table-require", "kr_req.txt", "--king-table-subset", "kr_sub.txt", "--parallel", "1", "2"], 63, "Error: --king-table-subset with --parallel is not supported by plink2_b200 yet."),
        (REQ + ["--king-table-require", "kr_req.txt", "--gpus", "2"], 63, "Error: --king-table-require[-xor] runs on one GPU; --gpus 2 is not supported with it."),
        (REQ + ["--king-table-require", "x_keep1.txt"], 7, "Error: No sample ID(s) in --king-table-require[-xor] file(s) are in the current\ndataset."),
        (REQ + ["--king-table-require-xor", "kr_req_allbut1.txt", "kr.fam"], 7, "Error: All sample ID(s) in --king-table-require-xor file(s) are in the current\ndataset."),
        (REQ + ["--king-table-require", "no_such_file.txt"], 3, "no_such_file.txt"),
    ],
)
def test_flag_checks(mock_so, tmp_path, args, code, msg):
    r = _run(mock_so, args, str(tmp_path / "o"), devices=2)
    assert r.returncode == code, r.stdout + r.stderr
    assert msg in r.stdout + r.stderr
