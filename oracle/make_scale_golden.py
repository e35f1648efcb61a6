#!/usr/bin/env python
"""Writes tests/golden/scale_reference.json and tests/golden/scale_grm_sample.npy: what the unmodified reference
(oracle/_ref/plink2[_lapack], oracle/build_ref.sh) outputs on the seeded filesets of oracle/synth.py, for the
at-scale parity tests of tests/test_scale_gpu.py.  Byte-exact outputs are stored as SHA-256 digests, the fp32 GRM as
a seeded sample of its entries.  Rerun only when the inputs or the commands of those tests change."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.synth import write_bed  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "plink2")
REF_LAPACK = os.path.join(ROOT, "oracle", "_ref", "plink2_lapack")
GOLDEN = os.path.join(ROOT, "tests", "golden")
THREADS = str(len(os.sched_getaffinity(0)))
GRM_SAMPLE, GRM_SAMPLE_SEED = 20_000, 7
# (samples, variants, seed) of each fileset; the tests generate the same ones
SETS = {"d4k": (4096, 65536, 1), "d20k": (20000, 2048, 5), "d3k": (3000, 4096, 9)}


def sha256(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for chunk in iter(lambda: f.read(1 << 24), b""):
            h.update(chunk)
    return h.hexdigest()


def run(cmd):
    subprocess.run(cmd + ["--threads", THREADS], check=True, stdout=subprocess.DEVNULL)


def main():
    out = {"sets": {k: list(v) for k, v in SETS.items()}}
    with tempfile.TemporaryDirectory() as d:
        pre = {k: os.path.join(d, k) for k in SETS}
        for k, (n, m, seed) in SETS.items():
            write_bed(pre[k], n, m, seed)
        r = os.path.join(d, "r")
        # KING 4096 x 65536: fp32 triangle + a table filtered at the 97 % quantile of the kinships
        run([REF, "--bfile", pre["d4k"], "--make-king", "bin4", "triangle", "--out", r])
        kin = np.fromfile(r + ".king.bin", dtype=np.float32)
        thr = repr(float(np.quantile(kin.astype(np.float64), 0.97)))
        run([REF, "--bfile", pre["d4k"], "--make-king-table", "counts", "cols=+ibs1,+ibs", "--king-table-filter", thr, "--out", r])
        out["king4k"] = {"filter": thr, "kin0_rows": sum(1 for _ in open(r + ".kin0")) - 1,
                         "sha256": {e: sha256(r + e) for e in (".king.bin", ".king.id", ".kin0")}}
        # KING 20000 x 2048: the whole triangle
        run([REF, "--bfile", pre["d20k"], "--make-king", "bin4", "triangle", "--out", r + "20k"])
        out["king20k"] = {"sha256": {".king.bin": sha256(r + "20k.king.bin")}}
        # KING 3000 x 4096 (multipass test)
        run([REF, "--bfile", pre["d3k"], "--make-king", "bin", "triangle", "--make-king-table", "counts", "--king-table-filter", "-0.05", "--out", r + "3k"])
        out["king3k"] = {"sha256": {e: sha256(r + "3k" + e) for e in (".king.bin", ".kin0")}}
        # GRM 4096 x 65536 (LAPACK build): exact .grm.N.bin / .grm.id, a seeded sample of the fp32 .grm.bin
        run([REF_LAPACK, "--bfile", pre["d4k"], "--make-grm-bin", "--out", r + "grm"])
        g = np.fromfile(r + "grm.grm.bin", dtype=np.float32)
        idx = np.sort(np.random.default_rng(GRM_SAMPLE_SEED).choice(g.size, GRM_SAMPLE, replace=False))
        np.save(os.path.join(GOLDEN, "scale_grm_sample.npy"), g[idx])
        out["grm4k"] = {"entries": int(g.size), "sample": GRM_SAMPLE, "sample_seed": GRM_SAMPLE_SEED,
                        "sha256": {e: sha256(r + "grm" + e) for e in (".grm.N.bin", ".grm.id")}}
        # --indep-pairwise 500 50 0.2 on the 4096 x 65536 set
        run([REF, "--bfile", pre["d4k"], "--indep-pairwise", "500", "50", "0.2", "--out", r + "ld"])
        out["prune4k"] = {"kept": sum(1 for _ in open(r + "ld.prune.in")),
                          "sha256": {e: sha256(r + "ld" + e) for e in (".prune.in", ".prune.out")}}
    with open(os.path.join(GOLDEN, "scale_reference.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
