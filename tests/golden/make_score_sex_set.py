#!/usr/bin/env python
"""Builds the sex-chromosome `--score` / `--variant-score` fixture for set X and records the reference's reports.

`x_score_sex.txt.gz` scores about half of set X's variants on every chromosome (1, X, Y, XY, MT), each by its REF or
its ALT allele at random; every 9th scored variant is named by both alleles, and a few lines carry unknown IDs or
foreign allele codes.  Three coefficient columns: BETA, NEG (negated and rescaled) and MIX (random signs).
`x_vscore_sex.txt` gives every sample of set X two weight columns.

Set X has unknown-sex samples, so the reference refuses mean imputation with chrY entries on the full set: the reports
with mean imputation run under `--remove-nosex`.  Every report is written under both `--xchr-model 2` (the default)
and `--xchr-model 1` where the model matters.  Scores are stored gzipped (both programs read gzipped inputs); the
reference runs on the plain files.
usage: make_score_sex_set.py <reference plink2> <golden dir>"""
import gzip
import os
import random
import shutil
import subprocess
import sys
import tempfile

SCORE = "x_score_sex.txt"
VSCORE = "x_vscore_sex.txt"
COLS = ["--score-col-nums", "3-5"]
FULL = ["cols=+scoresums,+denom,+dosagesum"]
RUNS = {
    "x_ssx_nmi": ["--score", SCORE, "header-read", "no-mean-imputation"] + FULL + COLS,
    "x_ssx_nmi1": ["--score", SCORE, "header-read", "no-mean-imputation"] + FULL + COLS + ["--xchr-model", "1"],
    "x_ssx_rn": ["--remove-nosex", "--score", SCORE, "header-read"] + FULL + COLS,
    "x_ssx_rn1": ["--remove-nosex", "--score", SCORE, "header-read"] + FULL + COLS + ["--xchr-model", "1"],
    "x_ssx_ctr1": ["--remove-nosex", "--score", SCORE, "header-read", "center", "cols=+scoresums"] + COLS + ["--xchr-model", "1"],
    "x_ssx_one": ["--score", SCORE, "1", "2", "4", "header-read", "no-mean-imputation", "cols=+denom,+dosagesum", "--xchr-model", "1"],
}
VRUNS = {
    "x_vsx": ["--remove-nosex", "--variant-score", VSCORE, "cols=+altfreq"],
    "x_vsx1": ["--remove-nosex", "--variant-score", VSCORE, "cols=+altfreq", "--xchr-model", "1"],
}


def write_inputs(gdir, tmp):
    bim = [ln.split() for ln in open(os.path.join(gdir, "x.bim"))]
    rng = random.Random(23)
    lines = []
    for k, (_, snp, _, _, a1, a2) in enumerate(bim):
        if rng.random() < 0.5:
            continue
        named = [rng.choice((a1, a2))]
        if len(lines) % 9 == 4:
            named = [a1, a2]
        for a in named:
            b = rng.uniform(-0.5, 0.5)
            lines.append([snp, a, "%.5g" % b, "%.5g" % (-1.3 * b), "%.5g" % (rng.choice((-1, 1)) * rng.uniform(0.01, 0.3))])
    for k in range(0, len(lines), 37):
        lines.insert(k, ["nosuch%d" % k, "A", "0.1", "0.2", "0.3"] if k % 2 else [lines[k][0], "Z", "0.1", "0.2", "0.3"])
    with open(os.path.join(tmp, SCORE), "w") as f:
        f.write("SNP\tA1\tBETA\tNEG\tMIX\n")
        for t in lines:
            f.write("\t".join(t) + "\n")
    with open(os.path.join(tmp, VSCORE), "w") as f:
        f.write("#FID\tIID\tV1\tV2\n")
        for ln in open(os.path.join(gdir, "x.fam")):
            t = ln.split()
            f.write("%s\t%s\t%.4g\t%.4g\n" % (t[0], t[1], rng.uniform(-1, 1), rng.choice((0.0, 0.5, 1.0, 2.5))))


def main():
    ref, gdir = (os.path.abspath(a) for a in sys.argv[1:3])
    tmp = tempfile.mkdtemp()
    try:
        write_inputs(gdir, tmp)
        for ext in ("bed", "bim", "fam"):
            shutil.copy(os.path.join(gdir, "x." + ext), tmp)

        def run(args, out):
            subprocess.run([ref, "--bfile", "x"] + args + ["--threads", "2", "--out", out], cwd=tmp, check=True, stdout=subprocess.DEVNULL)

        def keep(name, gz=True):
            with open(os.path.join(tmp, name), "rb") as f:
                data = f.read()
            if gz:
                with open(os.path.join(gdir, name + ".gz"), "wb") as o:
                    o.write(gzip.compress(data, mtime=0))
            else:
                with open(os.path.join(gdir, name), "wb") as o:
                    o.write(data)

        keep(SCORE)
        keep(VSCORE, gz=False)
        for name, args in RUNS.items():
            run(args, name)
            keep(name + ".sscore")
        for name, args in VRUNS.items():
            run(args, name)
            keep(name + ".vscore")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
