"""CPU: every shape and encoding of the --make-king and --make-rel matrices through the host program's writers, replayed
without a GPU on the stand-in library (tests/harness/mock_pl2gpu.cc, injected with LD_PRELOAD) and compared with the
files the reference wrote for set A (tests/golden/make_matrix_shapes_set.py).  KING matrices and text REL matrices are
byte-identical; the fp64 .rel.bin values differ from the reference's in the last bits only, because the stand-in sums
in another order."""
import gzip
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")

# (name, arguments, matrix file extension)
CASES = [
    ("king_sq0", ["--make-king", "square0"], ".king"),
    ("king_tri", ["--make-king", "triangle"], ".king"),
    ("king_bin_sq0", ["--make-king", "bin", "square0"], ".king.bin"),
    ("king_bin4_sq", ["--make-king", "bin4", "square"], ".king.bin"),
    ("king_bin_tri", ["--make-king", "bin", "triangle"], ".king.bin"),
    ("rel_tri", ["--make-rel", "triangle"], ".rel"),
    ("rel_sq0", ["--make-rel", "square0"], ".rel"),
    ("rel_bin_sq0", ["--make-rel", "bin", "square0"], ".rel.bin"),
    ("rel_bin4_sq", ["--make-rel", "bin4", "square"], ".rel.bin"),
    ("rel_bin_tri", ["--make-rel", "bin", "triangle"], ".rel.bin"),
    ("rel_cov_sq0", ["--make-rel", "cov", "square0"], ".rel"),
]


@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mock") / "mock_pl2gpu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", "mock_pl2gpu.cc")], check=True)
    return so


def _f64_close(got_bytes, ref_bytes):
    got = np.frombuffer(got_bytes, dtype=np.float64)
    ref = np.frombuffer(ref_bytes, dtype=np.float64)
    assert got.shape == ref.shape
    assert np.all(np.abs(got - ref) <= 1e-11 * np.abs(ref) + 1e-14)


@pytest.mark.parametrize("name,args,ext", CASES, ids=[c[0] for c in CASES])
def test_matrix_shape_matches_reference(mock_so, tmp_path, name, args, ext):
    out = str(tmp_path / "o")
    r = subprocess.run([BIN, "--bfile", "a"] + args + ["--out", out], capture_output=True, text=True, env=dict(os.environ, LD_PRELOAD=mock_so), cwd=GD)
    assert r.returncode == 0, r.stdout + r.stderr
    got = open(out + ext, "rb").read()
    ref = gzip.open(os.path.join(GD, "a_ms_%s%s.gz" % (name, ext)), "rb").read()
    if ext == ".rel.bin" and "bin4" not in args:
        _f64_close(got, ref)
    else:
        assert got == ref
    ids = ext.split(".")[1]
    assert open(out + "." + ids + ".id", "rb").read() == open(os.path.join(GD, "a_kingsq.king.id"), "rb").read()
