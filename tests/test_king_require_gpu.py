"""GPU: `--king-table-require[-xor]` on the KING tensor tile path.  The mapped job (pl2gpu_king_begin_mapped: samples
permuted into a device order on the device, tiles cut at a column bound) is checked bit-exact against the numpy
popcount restatement and against the pair-list kernel, for required sets that are contiguous, scattered or sit on tile
boundaries, with the non-required count n0 at every residue mod 128 where a row or column tile edge could go wrong
and variant counts that are not multiples of 256; the identity order must equal pl2gpu_king_begin_ex.  Through the
command line, every table of set KR must be byte-identical to the reference's, also when --gpu-memory splits the
slab into several passes."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from plink_ng_b200.host import KingJob, KingPairJob, MappedKingJob, pack_genotypes
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
GOLD = json.load(open(os.path.join(GD, "kr_digests.json")))


def _random_geno(m, n, seed, miss=0.03):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.02, 0.98, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _required(n, r, layout, seed):
    rng = np.random.default_rng(seed)
    if layout == "contiguous":
        req = np.arange(n - r, n)
    elif layout == "scattered":
        req = np.sort(rng.choice(n, size=r, replace=False))
    else:  # around multiples of 128 and 64
        edges = sorted({e + d for e in range(64, n, 64) for d in (-1, 0, 1) if 0 <= e + d < n})
        req = np.array(sorted(rng.choice(edges, size=min(r, len(edges)), replace=False)))
    return req


def _order(n, req):
    mask = np.zeros(n, dtype=bool)
    mask[req] = True
    return np.concatenate([np.flatnonzero(~mask), np.flatnonzero(mask)]).astype(np.uint32)


def _expected(geno, order, n0, col_end):
    """numpy popcount counts of the mapped slab: positions (j, i), n0 <= j < n, i < min(j, col_end), "1" = i."""
    g = geno[:, order]
    full = orc.king_counts(g, n0, g.shape[1])
    n = g.shape[1]
    keep = np.concatenate([np.arange(j) < col_end for j in range(n0, n)]) if n0 < n else np.zeros(0, dtype=bool)
    return full[keep]


N = 640


@pytest.mark.parametrize("n0_mod", [0, 1, 63, 64, 127, 128, 129])
@pytest.mark.parametrize("layout", ["contiguous", "scattered", "edges"])
@pytest.mark.parametrize("xor", [False, True])
def test_mapped_job_matches_popcount_and_pair_list(gpu_ctx, n0_mod, layout, xor):
    n0 = 256 + n0_mod
    m = 1000 + 37 * n0_mod  # never a multiple of 256
    geno = _random_geno(m, N, seed=n0 * 3 + len(layout))
    req = _required(N, N - n0, layout, seed=n0)
    order = _order(N, req)
    n0 = N - len(req)
    col_end = n0 if xor else N
    with MappedKingJob(gpu_ctx, N, order, n0, N, col_end, max_variants_per_add=512) as job:
        job.add_variants(pack_genotypes(geno))
        got = job.counts()
        kin = job.kinship()
    want = _expected(geno, order, n0, col_end)
    assert np.array_equal(got, want)
    pairs = np.array([(order[i], order[j]) for j in range(n0, N) for i in range(min(j, col_end))], dtype=np.uint32)
    with KingPairJob(gpu_ctx, N, pairs) as pj:
        pj.add_variants(pack_genotypes(geno))
        assert np.array_equal(pj.counts(), got)
    c = got.astype(np.float64)
    ref_kin = 0.5 - (4 * c[:, 0] + c[:, 2] + c[:, 3]) / (4 * (c[:, 1] + np.minimum(c[:, 2], c[:, 3])))
    assert np.array_equal(np.isnan(kin), np.isnan(ref_kin)) and np.allclose(kin[~np.isnan(kin)], ref_kin[~np.isnan(ref_kin)], rtol=0, atol=1e-15)


@pytest.mark.parametrize("xor", [False, True])
def test_mapped_filter_and_row_passes(gpu_ctx, xor):
    """get_filtered returns only pairs below the column bound; two row passes give the one-pass counts."""
    geno = _random_geno(777, N, seed=5)
    geno[:, 600] = geno[:, 10]  # a duplicate: kinship 0.5
    req = _required(N, 150, "scattered", seed=9)
    order = _order(N, req)
    n0 = N - len(req)
    col_end = n0 if xor else N
    want = _expected(geno, order, n0, col_end)
    mid = n0 + 70
    parts = []
    for r0, r1 in ((n0, mid), (mid, N)):
        with MappedKingJob(gpu_ctx, N, order, r0, r1, col_end) as job:
            job.add_variants(pack_genotypes(geno))
            parts.append(job.counts())
            pairs, counts, kin = job.filtered(-1.0)
            assert pairs.shape[0] == parts[-1].shape[0] and np.all(pairs[:, 1] < col_end) and np.all(pairs[:, 0] >= r0)
            assert np.array_equal(counts, parts[-1])
    assert np.array_equal(np.concatenate(parts), want)


@pytest.mark.parametrize("n", [2, 65, 641])
def test_identity_order_equals_begin_ex(gpu_ctx, n):
    geno = _random_geno(1300, n, seed=n)
    with KingJob(gpu_ctx, n) as job:
        job.add_variants(pack_genotypes(geno))
        want = job.counts()
    for order in (None, np.arange(n, dtype=np.uint32)):
        with MappedKingJob(gpu_ctx, n, order) as job:
            job.add_variants(pack_genotypes(geno))
            assert np.array_equal(job.counts(), want)


def _run(args, out):
    r = subprocess.run([BIN] + args + ["--out", out], capture_output=True, text=True, cwd=GD)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


@pytest.mark.parametrize("name", sorted(GOLD["runs"]))
def test_cli_matches_reference(tmp_path, name):
    out = str(tmp_path / "o")
    _run(GOLD["runs"][name], out)
    assert hashlib.sha256(open(out + ".kin0", "rb").read()).hexdigest() == GOLD["digests"][name]["sha256"]


def _write_bed(prefix, geno, ids):
    m, n = geno.shape
    code = np.array([0, 2, 3, 1], dtype=np.uint8)[geno]
    nb = (n + 3) // 4
    pad = np.zeros((m, nb * 4), dtype=np.uint8)
    pad[:, :n] = code
    packed = (pad[:, 0::4] | (pad[:, 1::4] << 2) | (pad[:, 2::4] << 4) | (pad[:, 3::4] << 6)).astype(np.uint8)
    with open(prefix + ".bed", "wb") as f:
        f.write(bytes([0x6C, 0x1B, 0x01]) + packed.tobytes())
    with open(prefix + ".bim", "w") as f:
        f.writelines("1\tv%d\t0\t%d\tA\tG\n" % (v, v + 1) for v in range(m))
    with open(prefix + ".fam", "w") as f:
        f.writelines("%s %s 0 0 1 -9\n" % x for x in ids)


@pytest.mark.parametrize("flag", ["--king-table-require", "--king-table-require-xor"])
def test_cli_multipass_equals_one_pass(tmp_path, flag):
    """5,000 samples, 2,000 of them required: --gpu-memory 600 forces several row passes over the variants."""
    n = 5000
    rng = np.random.default_rng(11)
    ids = [("F%d" % (k % 97), "s%03d" % k) for k in rng.permutation(n)]
    _write_bed(str(tmp_path / "d"), _random_geno(1500, n, seed=3), ids)
    with open(tmp_path / "req.txt", "w") as f:
        f.writelines("%s %s\n" % ids[k] for k in rng.choice(n, size=2000, replace=False))
    base = ["--bfile", str(tmp_path / "d"), "--make-king-table", "counts", "cols=+ibs1", flag, str(tmp_path / "req.txt")]
    one = _run(base, str(tmp_path / "one"))
    multi = _run(base + ["--gpu-memory", "600"], str(tmp_path / "multi"))
    assert "passes over the variants" not in one and "passes over the variants" in multi
    assert open(tmp_path / "one.kin0", "rb").read() == open(tmp_path / "multi.kin0", "rb").read()
