"""GPU: parity AT SCALE, through the product (the plink2_b200 host program), against what the UNMODIFIED reference
binary (oracle/_ref/plink2[_lapack]) wrote for the same seeded filesets (oracle/synth.py).  The reference's
outputs are stored under tests/golden/ by oracle/make_scale_golden.py: SHA-256 digests of every byte-exact file
and a seeded sample of the fp32 GRM.

Sizes are the ones SURVEY.md 8(c) names for the smoke set: 4,096 samples x 65,536 variants (32 row tiles x
up to 52 column tiles, two 32,768-variant batches for GRM / several for KING), plus a 20,000-sample KING
run (157 row tiles) that pins tile placement and orientation pair by pair, and a forced multipass run.
"""
import hashlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
ENV = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "scale_reference.json")))
sys.path.insert(0, ROOT)
from oracle.synth import write_bed  # noqa: E402


def sh(cmd, env=None, ok=(0,)):
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode in ok, " ".join(cmd) + "\n" + r.stdout[-2000:] + r.stderr[-2000:]
    return r


def sha256(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for chunk in iter(lambda: f.read(1 << 24), b""):
            h.update(chunk)
    return h.hexdigest()


def assert_same_as_reference(prefix, digests):
    """Every file prefix + ext byte-identical to the reference's (SHA-256 of the reference's file)."""
    bad = [ext for ext, want in digests.items() if sha256(prefix + ext) != want]
    assert not bad, f"differ from the reference's output: {', '.join(prefix + e for e in bad)}"


def fileset(tmp_path, name):
    pre = str(tmp_path / name)
    write_bed(pre, *GOLD["sets"][name])
    return pre


@pytest.fixture(scope="module")
def dummy4k(tmp_path_factory):
    return fileset(tmp_path_factory.mktemp("scale4k"), "d4k")


def test_king_table_and_matrix_4096x65536_byte_identical(dummy4k, tmp_path):
    """Every .kin0 count column (NSNP HETHET IBS0 HET1_HOM2 HET2_HOM1 IBS KINSHIP) on a NON-EMPTY filtered table
    (>= 1e5 rows; the filter is the 97 % quantile of the reference's kinships) plus the whole fp32 kinship triangle,
    byte for byte."""
    gold = GOLD["king4k"]
    out = str(tmp_path / "b200")
    flags = ["--make-king-table", "counts", "cols=+ibs1,+ibs", "--king-table-filter", gold["filter"]]
    sh([BIN, "--bfile", dummy4k] + flags + ["--make-king", "bin4", "triangle", "--out", out], env=ENV)
    assert gold["kin0_rows"] >= 100_000
    assert os.path.getsize(out + ".king.bin") == 4 * (4096 * 4095 // 2)
    rows = sum(1 for _ in open(out + ".kin0")) - 1
    assert rows == gold["kin0_rows"], rows
    assert_same_as_reference(out, gold["sha256"])


def test_king_matrix_20000_samples_pairwise(tmp_path):
    """157 row tiles x up to 250 column tiles: the whole 2e8-pair fp32 kinship triangle against the reference's, so a
    tile-placement or orientation error anywhere in the triangle fails (the marginal-sum test cannot see those)."""
    pre, out = fileset(tmp_path, "d20k"), str(tmp_path / "b200")
    sh([BIN, "--bfile", pre, "--make-king", "bin4", "triangle", "--out", out], env=ENV)
    assert os.path.getsize(out + ".king.bin") == 4 * (20000 * 19999 // 2)
    assert_same_as_reference(out, GOLD["king20k"]["sha256"])


def test_king_forced_multipass_matches_single_pass(tmp_path):
    """--gpu-memory caps the device budget so RunKing needs >= 3 row-block passes (the reference's
    CountTrianglePasses behaviour, 2.0/plink2_matrix_calc.cc:216-255); outputs must not change."""
    pre, one = fileset(tmp_path, "d3k"), str(tmp_path / "one")
    digests = GOLD["king3k"]["sha256"]
    flags = ["--make-king", "bin", "triangle", "--make-king-table", "counts", "--king-table-filter", "-0.05"]
    sh([BIN, "--bfile", pre] + flags + ["--out", one], env=ENV)
    assert_same_as_reference(one, digests)
    passes = 0
    for mib in (640, 560, 500, 470, 450, 435, 425, 415):
        multi = str(tmp_path / f"multi{mib}")
        r = sh([BIN, "--bfile", pre] + flags + ["--gpu-memory", str(mib), "--out", multi], env=ENV, ok=(0, 2))
        if r.returncode:
            break  # below the fixed staging buffers: nothing smaller can work
        m = re.search(r"(\d+) passes over the variants", r.stdout)
        passes = int(m.group(1)) if m else 1
        assert_same_as_reference(multi, digests)
        if passes >= 3:
            break
    assert passes >= 3, f"no --gpu-memory value produced >= 3 passes (last: {passes})"


def test_grm_4096x65536_vs_reference_blas(dummy4k, tmp_path):
    """.grm.bin against the LAPACK build of the reference (threaded OpenBLAS dsyrk in fp64) within 1e-5 relative on a
    seeded sample of 20,000 entries, .grm.N.bin (per-pair observation counts) and .grm.id exactly."""
    gold = GOLD["grm4k"]
    out = str(tmp_path / "b200")
    sh([BIN, "--bfile", dummy4k, "--make-grm-bin", "--out", out], env=ENV)
    b = np.fromfile(out + ".grm.bin", dtype=np.float32).astype(np.float64)
    assert b.size == gold["entries"] == 4096 * 4097 // 2
    idx = np.sort(np.random.default_rng(gold["sample_seed"]).choice(b.size, gold["sample"], replace=False))
    a = np.load(os.path.join(ROOT, "tests", "golden", "scale_grm_sample.npy")).astype(np.float64)
    # fp32 payload: half an ulp of the stored value (6e-8 relative) on top of the 1e-5 relative contract
    assert np.allclose(b[idx], a, rtol=1e-5, atol=2e-8), float(np.max(np.abs(a - b[idx])))
    assert_same_as_reference(out, gold["sha256"])


def test_indep_pairwise_500_50_02_keep_list_4096x65536(dummy4k, tmp_path):
    """The BASELINE config-4 command on the 65,536-variant set: .prune.in / .prune.out byte-identical."""
    gold = GOLD["prune4k"]
    out = str(tmp_path / "b200")
    sh([BIN, "--bfile", dummy4k, "--indep-pairwise", "500", "50", "0.2", "--out", out], env=ENV)
    assert 10_000 < gold["kept"] < 60_000, gold["kept"]
    assert sum(1 for _ in open(out + ".prune.in")) == gold["kept"]
    assert_same_as_reference(out, gold["sha256"])
