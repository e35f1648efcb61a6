#!/usr/bin/env python
"""Builds the `--q-score-range` fixtures for sets A and X and records the reference's reports for them.

Range files:
  `a_qsr_nested.ranges`  PRSice-style thresholds 0-0.001 .. 0-1, plus lines the reference skips (a non-numeric bound,
                         too few tokens);
  `a_qsr_mixed.ranges`   overlapping (lo / mid), disjoint (lo / hi) ranges, a point range (pt: 0.25 - 0.25) and a
                         range no variant lies in (none);
  `x_qsr.ranges`         three nested thresholds and a disjoint upper range.
Data files (variant ID, p-value):
  `a_qsr.pvals`          header line, IDs and p-values of most variants of set A: some `NA`, a few exactly 0.25, some
                         unknown IDs (skipped and counted);
  `a_qsr_min.pvals`      columns P, X, SNP (read as `3 1`) with a header; every 7th variant listed twice at different
                         p-values (for 'min');
  `x_qsr.pvals`          every variant of set X (chromosomes 1, X, Y, XY, MT), some `NA`.
The score files are the ones of make_score_cols_set.py (`a_score_cols.txt`) and make_score_sex_set.py
(`x_score_sex.txt`).  Every `<run>.<range>.sscore` the reference writes for RUNS is stored gzipped; a `zs` run's
`.sscore.zst` is stored decompressed and gzipped; `a_qsr_lv.sscore.vars` is the variant list of the `list-variants`
run.  The reference runs on the plain files.
usage: make_qsr_set.py <reference plink2> <golden dir>"""
import ctypes as C
import glob
import gzip
import os
import random
import shutil
import subprocess
import sys
import tempfile

A_SCORE = "a_score_cols.txt"
X_SCORE = "x_score_sex.txt"
NESTED = ["--q-score-range", "a_qsr_nested.ranges", "a_qsr.pvals", "header"]
MIXED = ["--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "header"]
X_QSR = ["--q-score-range", "x_qsr.ranges", "x_qsr.pvals"]
X_FULL = ["header-read", "cols=+scoresums,+denom,+dosagesum", "--score-col-nums", "3-5"]
RUNS = {
    "a_qsr_nest": ["--bfile", "a", "--score", A_SCORE, "1", "2", "3", "header"] + NESTED,
    "a_qsr_mix": ["--bfile", "a", "--score", A_SCORE, "header-read", "cols=+scoresums"] + MIXED,
    "a_qsr_min": ["--bfile", "a", "--score", A_SCORE, "header", "--q-score-range", "a_qsr_mixed.ranges", "a_qsr_min.pvals", "3", "1", "header", "min"],
    "a_qsr_cols": ["--bfile", "a", "--score", A_SCORE, "header-read", "--score-col-nums", "3-7"] + NESTED,
    "a_qsr_vs": ["--bfile", "a", "--score", A_SCORE, "header-read", "variance-standardize", "cols=+scoresums", "--score-col-nums", "3-7"] + MIXED,
    "a_qsr_nmi": ["--bfile", "a", "--score", A_SCORE, "header-read", "no-mean-imputation", "cols=+denom,+dosagesum,+scoresums", "--score-col-nums", "3-7"] + MIXED,
    "a_qsr_zs": ["--bfile", "a", "--score", A_SCORE, "header-read", "zs"] + NESTED,
    "a_qsr_lv": ["--bfile", "a", "--score", A_SCORE, "header-read", "list-variants"] + MIXED,
    "x_qsr_rn1": ["--bfile", "x", "--remove-nosex", "--score", X_SCORE] + X_FULL + ["--xchr-model", "1"] + X_QSR,
    "x_qsr_rn2": ["--bfile", "x", "--remove-nosex", "--score", X_SCORE] + X_FULL + ["--xchr-model", "2"] + X_QSR,
    "x_qsr_nmi1": ["--bfile", "x", "--score", X_SCORE, "no-mean-imputation"] + X_FULL + ["--xchr-model", "1"] + X_QSR,
}


def write_inputs(gdir, tmp):
    def out(name, lines):
        with open(os.path.join(gdir, name), "w") as f:
            f.write("".join(ln + "\n" for ln in lines))

    out("a_qsr_nested.ranges", ["S1 0 0.001", "S2 0 0.01", "bad x 0.5", "S3 0 0.05", "S4 0 0.1", "short 0.2", "S5 0 0.5", "S6 0 1"])
    out("a_qsr_mixed.ranges", ["lo 0 0.2", "mid 0.15 0.6", "hi 0.6 1", "pt 0.25 0.25", "none 2 3"])
    out("x_qsr.ranges", ["T1 0 0.05", "T2 0 0.3", "T3 0 1", "U 0.5 1"])
    rng = random.Random(41)
    a_ids = [ln.split()[1] for ln in open(os.path.join(gdir, "a.bim"))]
    lines = ["SNP\tP"]
    for k, snp in enumerate(a_ids):
        u = rng.random()
        if u < 0.05:
            continue
        p = "NA" if u < 0.09 else "0.25" if u < 0.12 else "%.4g" % (rng.random() ** 3)
        lines.append("%s\t%s" % (snp, p))
        if k % 97 == 3:
            lines.append("unknown%d\t0.01" % k)
    out("a_qsr.pvals", lines)
    lines = ["P\tX\tSNP"]
    for k, snp in enumerate(a_ids):
        p = rng.random() ** 2
        lines.append("%.4g\t.\t%s" % (p, snp))
        if k % 7 == 2:
            lines.append("%.4g\t.\t%s" % (rng.random(), snp))
    out("a_qsr_min.pvals", lines)
    lines = []
    for ln in open(os.path.join(gdir, "x.bim")):
        u = rng.random()
        lines.append("%s %s" % (ln.split()[1], "NA" if u < 0.05 else "%.4g" % rng.random()))
    out("x_qsr.pvals", lines)
    for name in (A_SCORE, X_SCORE):
        with gzip.open(os.path.join(gdir, name + ".gz"), "rb") as f, open(os.path.join(tmp, name), "wb") as o:
            o.write(f.read())
    for name in ("a_qsr_nested.ranges", "a_qsr_mixed.ranges", "x_qsr.ranges", "a_qsr.pvals", "a_qsr_min.pvals", "x_qsr.pvals"):
        shutil.copy(os.path.join(gdir, name), tmp)
    for s in ("a", "x"):
        for ext in ("bed", "bim", "fam"):
            shutil.copy(os.path.join(gdir, s + "." + ext), tmp)


def zstd_decompress(raw):
    z = C.CDLL("libzstd.so.1")
    z.ZSTD_findFrameCompressedSize.restype = C.c_size_t
    z.ZSTD_findFrameCompressedSize.argtypes = [C.c_void_p, C.c_size_t]
    z.ZSTD_getFrameContentSize.restype = C.c_ulonglong
    z.ZSTD_getFrameContentSize.argtypes = [C.c_void_p, C.c_size_t]
    z.ZSTD_decompress.restype = C.c_size_t
    z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    buf = C.create_string_buffer(raw, len(raw))
    base = C.addressof(buf)
    out, off = b"", 0
    while off < len(raw):
        fsz = z.ZSTD_findFrameCompressedSize(base + off, len(raw) - off)
        n = z.ZSTD_getFrameContentSize(base + off, fsz)
        dst = C.create_string_buffer(max(int(n), 1))
        assert z.ZSTD_decompress(dst, n, base + off, fsz) == n
        out += dst.raw[:n]
        off += fsz
    return out


def main():
    ref, gdir = (os.path.abspath(a) for a in sys.argv[1:3])
    tmp = tempfile.mkdtemp()
    try:
        write_inputs(gdir, tmp)
        for name, args in RUNS.items():
            subprocess.run([ref] + args + ["--threads", "2", "--out", name], cwd=tmp, check=True, stdout=subprocess.DEVNULL)
            for path in sorted(glob.glob(os.path.join(tmp, name + ".*.sscore*")) + glob.glob(os.path.join(tmp, name + ".sscore.vars"))):
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
