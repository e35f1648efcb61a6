#!/usr/bin/env python
"""Builds the several-column `--score` fixture for set A and records the reference's reports for it.

`a_score_cols.txt.gz` keeps the lines of `a_score.txt` (shuffled REF / ALT entries, unknown IDs, foreign allele codes, a
header line) and gives each five coefficient columns: BETA (the original), NEG (negated and rescaled), ZERO (all
zero), MIX (random signs) and HALF (BETA / 2).  Every 17th line has all five coefficients zero.

The reference's `.sscore` is stored for each command line in RUNS; the projection pair is the reference's
`--pca 10 allele-wts` (LAPACK build, variants with MAF >= 0.01: the reference refuses to variance-standardize a
monomorphic variant named by its REF allele) `.eigenvec.allele` and `.afreq` of set A, and the `.sscore` of scoring set
A against those allele weights as plink2's documentation does it.  `a_vsc.vscore` is `--variant-score` with
`--vscore-col-nums 3` (the second weight column of `a_vscore_weights.txt`).  Every file is stored gzipped (both
programs read gzipped inputs); the reference runs on the plain files.
usage: make_score_cols_set.py <reference plink2> <reference plink2_lapack> <golden dir>"""
import gzip
import os
import random
import shutil
import subprocess
import sys
import tempfile

SCORE = "a_score_cols.txt"
PC_SCORE = ["--score", "a_pcw.eigenvec.allele", "2", "6", "header-read", "no-mean-imputation", "variance-standardize", "--score-col-nums", "7-16", "--read-freq", "a_pcw.afreq"]
RUNS = {
    "a_scc": ["--bfile", "a", "--score", SCORE, "--score-col-nums", "3-7"],
    "a_scc_hr": ["--bfile", "a", "--score", SCORE, "header-read", "--score-col-nums", "3-7"],
    "a_scc_nmi": ["--bfile", "a", "--score", SCORE, "header-read", "no-mean-imputation", "cols=+scoresums,+denom", "--score-col-nums", "3-7"],
    "a_scc_vs": ["--bfile", "a", "--score", SCORE, "header-read", "variance-standardize", "cols=+scoresums", "--score-col-nums", "3-7"],
    "a_scc_dom": ["--bfile", "a", "--score", SCORE, "header-read", "dominant", "cols=+scoresums", "--score-col-nums", "3-7"],
    "a_scc_ord": ["--bfile", "a", "--score", SCORE, "header-read", "cols=+scoresums", "--score-col-nums", "6", "5-7,3"],
    "a_scc_pc": ["--bfile", "a"] + PC_SCORE,
}
VSCORE = ["--bfile", "a", "--variant-score", "a_vscore_weights.txt", "--vscore-col-nums", "3"]


def write_score_file(gdir, tmp):
    rows = [ln.split() for ln in open(os.path.join(gdir, "a_score.txt"))][1:]
    rng = random.Random(31)
    with open(os.path.join(tmp, SCORE), "w") as f:
        f.write("SNP\tA1\tBETA\tNEG\tZERO\tMIX\tHALF\n")
        for k, (snp, a1, beta) in enumerate(rows):
            b = float(beta)
            cols = [beta, "%.5g" % (-1.7 * b), "0", "%.5g" % (rng.choice((-1, 1)) * rng.uniform(0.01, 0.3)), "%.5g" % (b / 2)]
            if k % 17 == 5:
                cols = ["0"] * 5
            f.write("\t".join([snp, a1] + cols) + "\n")


def main():
    ref, ref_lapack, gdir = (os.path.abspath(a) for a in sys.argv[1:4])
    tmp = tempfile.mkdtemp()
    try:
        write_score_file(gdir, tmp)
        for ext in ("bed", "bim", "fam"):
            shutil.copy(os.path.join(gdir, "a." + ext), tmp)
        shutil.copy(os.path.join(gdir, "a_vscore_weights.txt"), tmp)

        def run(binary, args, out):
            subprocess.run([binary] + args + ["--threads", "2", "--out", out], cwd=tmp, check=True, stdout=subprocess.DEVNULL)

        def keep(name):
            with open(os.path.join(tmp, name), "rb") as f, open(os.path.join(gdir, name + ".gz"), "wb") as o:
                o.write(gzip.compress(f.read(), mtime=0))

        keep(SCORE)
        run(ref_lapack, ["--bfile", "a", "--maf", "0.01", "--freq", "--pca", "10", "allele-wts"], "a_pcw")
        keep("a_pcw.eigenvec.allele")
        keep("a_pcw.afreq")
        for name, args in RUNS.items():
            run(ref, args, name)
            keep(name + ".sscore")
        run(ref, VSCORE, "a_vsc")
        keep("a_vsc.vscore")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
