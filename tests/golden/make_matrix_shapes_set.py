#!/usr/bin/env python
"""Writes the reference's --make-king / --make-rel matrices over set A in the shapes and encodings the other fixtures
leave out (tests/test_matrix_shapes.py): square0 and triangle text, fp64 square0 and triangle, fp32 square, and the
covariance form of square0.  Every file is stored gzipped as a_ms_<case><ext>.gz.
usage (from the repository root): python tests/golden/make_matrix_shapes_set.py"""
import gzip
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from test_matrix_shapes import CASES  # noqa: E402

REF = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "plink2")

with tempfile.TemporaryDirectory() as tmp:
    for name, args, ext in CASES:
        out = os.path.join(tmp, name)
        subprocess.run([REF, "--bfile", "a"] + args + ["--threads", "2", "--out", out], cwd=HERE, check=True, stdout=subprocess.DEVNULL)
        with open(out + ext, "rb") as f, gzip.GzipFile(os.path.join(HERE, "a_ms_%s%s.gz" % (name, ext)), "wb", 9, mtime=0) as g:
            g.write(f.read())
