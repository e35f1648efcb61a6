#!/usr/bin/env python
"""Builds set KR, the `--king-table-require[-xor]` fixture, and records the reference's `.kin0` tables for it.

KR is 700 samples x 3,000 variants (3 % missing calls, seeded) in .bed/.bim/.fam, so the required pairs cross several
128-row and 64-column pair tiles.  The sample IDs are not in natural order: 37 families with mixed-case names, leading
zeros and digit runs, plus 40 samples of FID 0 that an IID-only list can name; 24 samples are noisy copies of others so
that `--king-table-filter` keeps some pairs.  Require lists: `kr_req.txt` (45 samples scattered over the file, header
`#FID IID`), the same split across `kr_req_b1.txt` (FID IID lines) and `kr_req_b2.txt` (IID only: the FID-0 samples),
`kr_req_one.txt` (one sample), `kr_req_allbut1.txt` (every sample but one, for -xor); `kr_sub.txt` is a
`--king-table-subset` file of 3,000 random pairs in random orientation; `a_req.txt` names 9 samples of set A.

Every table the reference writes for the command lines in RUNS is stored as its SHA-256 in `kr_digests.json`; tables
of at most 200 kB are stored as well, gzipped (`<name>.kin0.gz`).
usage: make_king_require_set.py <reference plink2> <golden dir>"""
import gzip
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

N, M = 700, 3000

RUNS = {
    "kr_req": ["--bfile", "kr", "--make-king-table", "counts", "cols=+ibs1,+ibs", "--king-table-require", "kr_req.txt"],
    "kr_xor": ["--bfile", "kr", "--make-king-table", "counts", "cols=+ibs1,+ibs", "--king-table-require-xor", "kr_req.txt"],
    "kr_reqp": ["--bfile", "kr", "--make-king-table", "--king-table-require", "kr_req.txt"],
    "kr_reqf": ["--bfile", "kr", "--make-king-table", "cols=+ibs1", "--king-table-filter", "0.05", "--king-table-require", "kr_req.txt"],
    "kr_xorf": ["--bfile", "kr", "--make-king-table", "cols=+ibs1", "--king-table-filter", "0.05", "--king-table-require-xor", "kr_req.txt"],
    "kr_req2": ["--bfile", "kr", "--make-king-table", "counts", "cols=+ibs1", "--king-table-require", "kr_req_b1.txt", "kr_req_b2.txt"],
    "kr_relreq": ["--bfile", "kr", "--make-king-table", "rel-check", "counts", "cols=+ibs1", "--king-table-require", "kr_req.txt"],
    "kr_subxor": ["--bfile", "kr", "--make-king-table", "counts", "cols=+ibs1", "--king-table-subset", "kr_sub.txt", "--king-table-require-xor", "kr_req.txt"],
    "kr_one": ["--bfile", "kr", "--make-king-table", "counts", "cols=+ibs1,+ibs", "--king-table-require", "kr_req_one.txt"],
    "kr_xorall": ["--bfile", "kr", "--make-king-table", "counts", "cols=+ibs1", "--king-table-require-xor", "kr_req_allbut1.txt"],
    "a_kreq": ["--bfile", "a", "--make-king-table", "counts", "cols=+ibs1,+ibs", "--king-table-require", "a_req.txt"],
    "a_kreqx": ["--bfile", "a", "--make-king-table", "--king-table-require-xor", "a_req.txt"],
}


def sample_ids(rng):
    fams = []
    for f in range(37):
        base = ["fam", "Fam", "FAM", "f", "F"][f % 5]
        num = str(rng.integers(1, 60))
        if f % 3 == 0:
            num = "0" + num
        fams.append(base + num)
    fams = list(dict.fromkeys(fams))
    ids, seen = [], set()
    while len(ids) < N - 40:
        fid = fams[rng.integers(len(fams))]
        iid = ["id", "ID", "Id", "s", "S"][rng.integers(5)] + ("0" * int(rng.integers(0, 3))) + str(rng.integers(1, 400))
        if (fid, iid) not in seen:
            seen.add((fid, iid))
            ids.append((fid, iid))
    zero = []
    while len(zero) < 40:
        iid = ["z", "Z"][rng.integers(2)] + ("0" * int(rng.integers(0, 2))) + str(rng.integers(1, 200))
        if ("0", iid) not in seen:
            seen.add(("0", iid))
            zero.append(("0", iid))
    # the FID-0 samples spread through the file
    for k, z in enumerate(zero):
        ids.insert(int(k * (N - 40) / 40) + k, z)
    return ids


def write_set(gd, rng):
    ids = sample_ids(rng)
    freq = rng.uniform(0.05, 0.95, size=M)
    g = (rng.random((M, N)) < freq[:, None]).astype(np.uint8) + (rng.random((M, N)) < freq[:, None]).astype(np.uint8)
    for k in range(24):  # noisy copies: close relatives for --king-table-filter
        src, dst = int(rng.integers(N)), int(rng.integers(N))
        if src == dst:
            continue
        keep = rng.random(M) < rng.uniform(0.4, 0.9)
        g[keep, dst] = g[keep, src]
    code = np.where(rng.random((M, N)) < 0.03, 3, g)  # 0 hom A1 (ALT), 1 het, 2 hom A2, 3 missing
    bed_code = np.array([0, 2, 3, 1], dtype=np.uint8)[code]  # PLINK 1 .bed: 00 hom A1, 10 het, 11 hom A2, 01 missing
    nb = (N + 3) // 4
    pad = np.zeros((M, nb * 4), dtype=np.uint8)
    pad[:, :N] = bed_code
    packed = (pad[:, 0::4] | (pad[:, 1::4] << 2) | (pad[:, 2::4] << 4) | (pad[:, 3::4] << 6)).astype(np.uint8)
    with open(os.path.join(gd, "kr.bed"), "wb") as f:
        f.write(bytes([0x6C, 0x1B, 0x01]))
        f.write(packed.tobytes())
    with open(os.path.join(gd, "kr.bim"), "w") as f:
        for v in range(M):
            f.write("%d\tkr%d\t0\t%d\tA\tG\n" % (1 + v // 1000, v, 1000 + 100 * v))
    with open(os.path.join(gd, "kr.fam"), "w") as f:
        for fid, iid in ids:
            f.write("%s %s 0 0 %d -9\n" % (fid, iid, 1 + int(rng.integers(2))))
    return ids


def write_lists(gd, ids, rng):
    req = sorted(set(int(x) for x in rng.choice(N, size=40, replace=False)) | {0, 127, 128, 640, 699})
    zero_req = [k for k in req if ids[k][0] == "0"]
    if not zero_req:  # the IID-only file must name someone
        zero_req = [next(k for k in range(N) if ids[k][0] == "0")]
        req = sorted(set(req) | set(zero_req))
    with open(os.path.join(gd, "kr_req.txt"), "w") as f:
        f.write("#FID\tIID\n")
        for k in req:
            f.write("%s\t%s\n" % ids[k])
    with open(os.path.join(gd, "kr_req_b1.txt"), "w") as f:
        for k in req:
            if k not in zero_req:
                f.write("%s %s\n" % ids[k])
    with open(os.path.join(gd, "kr_req_b2.txt"), "w") as f:
        for k in zero_req:
            f.write("%s\n" % ids[k][1])
    with open(os.path.join(gd, "kr_req_one.txt"), "w") as f:
        f.write("%s %s\n" % ids[333])
    with open(os.path.join(gd, "kr_req_allbut1.txt"), "w") as f:
        for k in range(N):
            if k != 411:
                f.write("%s %s\n" % ids[k])
    with open(os.path.join(gd, "kr_sub.txt"), "w") as f:
        f.write("#FID1\tID1\tFID2\tID2\n")
        for _ in range(3000):
            a, b = (int(x) for x in rng.choice(N, size=2, replace=False))
            f.write("%s\t%s\t%s\t%s\n" % (ids[a] + ids[b]))
    a_ids = [ln.split()[:2] for ln in open(os.path.join(gd, "a.fam"))]
    with open(os.path.join(gd, "a_req.txt"), "w") as f:
        for k in (3, 17, 40, 41, 63, 64, 65, 90, 99):
            f.write("%s %s\n" % tuple(a_ids[k]))


def main():
    ref, gd = os.path.abspath(sys.argv[1]), os.path.abspath(sys.argv[2])
    rng = np.random.default_rng(20261017)
    ids = write_set(gd, rng)
    write_lists(gd, ids, rng)
    digests = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, args in RUNS.items():
            out = os.path.join(tmp, name)
            subprocess.run([ref] + args + ["--threads", "4", "--out", out], cwd=gd, check=True, stdout=subprocess.DEVNULL)
            data = open(out + ".kin0", "rb").read()
            digests[name] = {"sha256": hashlib.sha256(data).hexdigest(), "lines": data.count(b"\n")}
            if len(data) <= 200_000:
                with gzip.GzipFile(os.path.join(gd, name + ".kin0.gz"), "wb", mtime=0) as f:
                    f.write(data)
    with open(os.path.join(gd, "kr_digests.json"), "w") as f:
        json.dump({"runs": RUNS, "digests": digests}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
