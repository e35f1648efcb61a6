#!/usr/bin/env python
"""Builds the `--score-list` fixtures for sets A and X and records the reference's reports for them.

Score files (each with a header line; pieces of a_score_cols.txt / x_score_sex.txt):
  `a_sl_1.txt`   entries 0 - 249 of a_score_cols.txt;
  `a_sl_2.txt`   entries 150 - 411 (overlaps a_sl_1.txt in 150 - 249);
  `a_sl_3.txt`   every second entry of 0 - 119 whose variant a_sl_2.txt does not name (disjoint from it), entries
                 160 - 239 (every 8th) naming the variant's other allele, and three IDs that are not in the dataset;
  `x_sl_1.txt`, `x_sl_2.txt`  entries 0 - 299 and 200 - 469 of x_score_sex.txt (every ploidy class of set X);
  `d_sl_1.txt`, `d_sl_2.txt`  all entries and entries 100 - 299 of a_score_cols.txt, scored against `d.bim`.
Lists:
  `a_sl.list`      a_sl_1.txt, a_sl_2.txt (indented, with a second token the reader ignores), a_sl_3.txt and
                   a_sl_1.txt again;
  `a_sl_one.list`  a_sl_2.txt alone;  `x_sl.list`  x_sl_1.txt, x_sl_2.txt;  `d_sl.list`  d_sl_1.txt, d_sl_2.txt.
`d.bim` is a.bim with the variant after each of 14 variants the score files name renamed to that variant's ID, so that
those IDs occur twice ('ignore-dup-ids'); its genotypes are a.bed / a.fam.  Every `<run>[.<range>].sscore` the reference writes for RUNS is
stored gzipped (a `zs` run's decompressed).  The reference runs on the plain files.
usage: make_score_list_set.py <reference plink2> <golden dir>"""
import glob
import gzip
import os
import shutil
import subprocess
import sys
import tempfile

from make_qsr_set import zstd_decompress

A_LIST = ["--bfile", "a", "--score-list", "a_sl.list"]
X_LIST = ["--score-list", "x_sl.list", "header-read", "cols=+scoresums"]
X_COLS = ["--score-col-nums", "3-5"]
D_SET = ["--bed", "a.bed", "--bim", "d.bim", "--fam", "a.fam"]
RUNS = {
    "a_sl_plain": A_LIST + ["header"],
    "a_sl_hr": A_LIST + ["header-read", "cols=+scoresums"],
    "a_sl_cols": A_LIST + ["header-read", "--score-col-nums", "3-7"],
    "a_sl_center": A_LIST + ["header-read", "center"],
    "a_sl_vs": A_LIST + ["header-read", "variance-standardize", "cols=+scoresums"],
    "a_sl_dom": A_LIST + ["header-read", "dominant"],
    "a_sl_rec": A_LIST + ["header-read", "recessive"],
    "a_sl_nmi": A_LIST + ["header-read", "no-mean-imputation", "cols=+scoresums", "--score-col-nums", "3,5"],
    "a_sl_zs": A_LIST + ["header", "zs"],
    "a_sl_rf": A_LIST + ["header-read", "--read-freq", "a_rf.afreq"],
    "a_sl_qsr": A_LIST + ["header-read", "cols=+scoresums", "--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "header"],
    "a_sl_one": ["--bfile", "a", "--score-list", "a_sl_one.list", "header-read"],
    "x_sl_rn1": ["--bfile", "x", "--remove-nosex"] + X_LIST + X_COLS + ["--xchr-model", "1"],
    "x_sl_rn2": ["--bfile", "x", "--remove-nosex"] + X_LIST + X_COLS + ["--xchr-model", "2"],
    "x_sl_nmi1": ["--bfile", "x"] + X_LIST + ["no-mean-imputation"] + X_COLS + ["--xchr-model", "1"],
    "d_dup_score": D_SET + ["--score", "d_sl_1.txt", "header", "ignore-dup-ids"],
    "d_dup_list": D_SET + ["--score-list", "d_sl.list", "header", "ignore-dup-ids", "cols=+scoresums"],
}
INPUTS = ["a_sl_1.txt", "a_sl_2.txt", "a_sl_3.txt", "x_sl_1.txt", "x_sl_2.txt", "d_sl_1.txt", "d_sl_2.txt", "a_sl.list", "a_sl_one.list", "x_sl.list", "d_sl.list", "d.bim"]


def write_inputs(gdir):
    def out(name, lines):
        with open(os.path.join(gdir, name), "w") as f:
            f.write("".join(ln + "\n" for ln in lines))

    a = gzip.open(os.path.join(gdir, "a_score_cols.txt.gz"), "rt").read().rstrip("\n").split("\n")
    x = gzip.open(os.path.join(gdir, "x_score_sex.txt.gz"), "rt").read().rstrip("\n").split("\n")
    ah, ae = a[0], a[1:]
    xh, xe = x[0], x[1:]
    bim = {t[1]: (t[5], t[4]) for t in (ln.split() for ln in open(os.path.join(gdir, "a.bim")))}
    out("a_sl_1.txt", [ah] + ae[:250])
    out("a_sl_2.txt", [ah] + ae[150:])
    in_second = {ln.split("\t")[0] for ln in ae[150:]}
    third = [ln for ln in ae[:120:2] if ln.split("\t")[0] not in in_second]
    named = {tuple(ln.split("\t")[:2]) for ln in third}
    for ln in ae[160:240:8]:
        t = ln.split("\t")
        ref, alt = bim[t[0]]
        t[1] = alt if t[1] == ref else ref
        if (t[0], t[1]) not in named:
            named.add((t[0], t[1]))
            third.append("\t".join(t))
    third += ["nosuch%d\tA\t0.5\t0.5\t0\t0.5\t0.25" % k for k in range(3)]
    out("a_sl_3.txt", [ah] + third)
    out("x_sl_1.txt", [xh] + xe[:300])
    out("x_sl_2.txt", [xh] + xe[200:])
    out("d_sl_1.txt", [ah] + ae)
    out("d_sl_2.txt", [ah] + ae[100:300])
    out("a_sl.list", ["a_sl_1.txt", "  a_sl_2.txt\tignored", "a_sl_3.txt", "a_sl_1.txt"])
    out("a_sl_one.list", ["a_sl_2.txt"])
    out("x_sl.list", ["x_sl_1.txt", "x_sl_2.txt"])
    out("d_sl.list", ["d_sl_1.txt", "d_sl_2.txt"])
    d = [ln.split("\t") for ln in open(os.path.join(gdir, "a.bim")).read().rstrip("\n").split("\n")]
    row = {t[1]: k for k, t in enumerate(d)}
    named = [row[t] for t in dict.fromkeys(ln.split("\t")[0] for ln in ae) if t in row]
    for k in named[:40:3]:
        d[(k + 1) % len(d)][1] = d[k][1]
    out("d.bim", ["\t".join(t) for t in d])


def main():
    ref, gdir = (os.path.abspath(a) for a in sys.argv[1:3])
    write_inputs(gdir)
    tmp = tempfile.mkdtemp()
    try:
        for name in INPUTS + ["a_qsr_mixed.ranges", "a_qsr.pvals", "a_rf.afreq"] + ["%s.%s" % (s, e) for s in "ax" for e in ("bed", "bim", "fam")]:
            shutil.copy(os.path.join(gdir, name), tmp)
        for name, args in RUNS.items():
            subprocess.run([ref] + args + ["--threads", "2", "--out", name], cwd=tmp, check=True, stdout=subprocess.DEVNULL)
            for path in sorted(glob.glob(os.path.join(tmp, name + ".sscore*")) + glob.glob(os.path.join(tmp, name + ".*.sscore*"))):
                data = open(path, "rb").read()
                base = os.path.basename(path)
                if base.endswith(".zst"):
                    data, base = zstd_decompress(data), base[:-4]
                with open(os.path.join(gdir, base + ".gz"), "wb") as o:
                    o.write(gzip.compress(data, mtime=0))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
