#!/usr/bin/env python
"""Writes the `--variant-score` edge fixtures of tests/test_pca_products_gpu.py into tests/golden/: a 3-sample
fileset (v3.bed/.bim/.fam) whose variants cover every genotype pattern that matters to the imputation (monomorphic,
all-missing, polymorphic with missing calls), a weight file (v3_w.txt), a --read-freq file (v3_rf.afreq) that gives
ALT frequencies of exactly 0 and 1 to polymorphic variants with missing calls, and what the unmodified reference
(oracle/_ref/plink2, oracle/build_ref.sh) writes for both runs (v3.vscore, v3_rf.vscore).  Rerun only when the
inputs change."""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "plink2")
GOLDEN = os.path.join(ROOT, "tests", "golden")

# ALT dosage per (variant, sample); 3 = missing
GENO = [
    (0, 1, 2),
    (2, 2, 2),  # monomorphic ALT
    (0, 0, 0),  # monomorphic REF
    (3, 3, 3),  # all missing: frequency 0.5
    (1, 3, 0),
    (3, 2, 1),
    (2, 3, 2),
    (0, 3, 0),
    (1, 1, 3),
    (3, 0, 2),
    (2, 1, 3),
    (0, 2, 3),
]
WEIGHTS = ("#FID\tIID\tW1\tW2\tW3\n"
           "f0\ti0\t1.5\t-2\t1048576.25\n"
           "f1\ti1\t0.25\t3\t-0.75\n"
           "f2\ti2\t-1\t0.5\t3.5\n")
# --read-freq ALT frequencies; variants not listed keep the dataset's own
READ_FREQ_ALT = {"v4": "0", "v5": "1", "v8": "0", "v10": "1", "v11": "0.25"}
_BED_CODE = np.array([3, 2, 0, 1], dtype=np.uint8)  # ALT dosage 0/1/2, missing -> .bed 2-bit code


def write_fileset(prefix):
    g = np.array(GENO, dtype=np.uint8)
    m, n = g.shape
    codes = np.concatenate([_BED_CODE[g], np.zeros((m, (-n) % 4), dtype=np.uint8)], axis=1).reshape(m, -1, 4)
    packed = (codes[..., 0] | (codes[..., 1] << 2) | (codes[..., 2] << 4) | (codes[..., 3] << 6)).astype(np.uint8)
    with open(prefix + ".bed", "wb") as f:
        f.write(bytes([0x6C, 0x1B, 0x01]) + packed.tobytes())
    with open(prefix + ".bim", "w") as f:
        f.write("".join(f"1\tv{k}\t0\t{10 * (k + 1)}\tA\tG\n" for k in range(m)))
    with open(prefix + ".fam", "w") as f:
        f.write("".join(f"f{k}\ti{k}\t0\t0\t{1 + k % 2}\t-9\n" for k in range(n)))


def run(args):
    subprocess.run([REF, *args, "--threads", "1"], check=True, stdout=subprocess.DEVNULL)


def main():
    pre = os.path.join(GOLDEN, "v3")
    write_fileset(pre)
    with open(pre + "_w.txt", "w") as f:
        f.write(WEIGHTS)
    with tempfile.TemporaryDirectory() as d:
        t = os.path.join(d, "t")
        run(["--bfile", pre, "--freq", "--out", t])
        lines = open(t + ".afreq").read().split("\n")
        col = {name: i for i, name in enumerate(lines[0].lstrip("#").split("\t"))}
        out = [lines[0]]
        for ln in lines[1:]:
            if ln:
                f = ln.split("\t")
                f[col["ALT_FREQS"]] = READ_FREQ_ALT.get(f[col["ID"]], f[col["ALT_FREQS"]])
                out.append("\t".join(f))
        with open(pre + "_rf.afreq", "w") as f:
            f.write("\n".join(out) + "\n")
        run(["--bfile", pre, "--variant-score", pre + "_w.txt", "--out", t + "a"])
        run(["--bfile", pre, "--read-freq", pre + "_rf.afreq", "--variant-score", pre + "_w.txt", "cols=+altfreq", "--out", t + "b"])
        for src, dst in ((t + "a.vscore", "v3.vscore"), (t + "b.vscore", "v3_rf.vscore")):
            with open(src) as fi, open(os.path.join(GOLDEN, dst), "w") as fo:
                fo.write(fi.read())


if __name__ == "__main__":
    sys.exit(main())
