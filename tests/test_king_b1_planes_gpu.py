"""GPU: the column plane copy the default KING kernel reads, and the tile pairs it runs as 2-CTA clusters.

The prep stream writes, next to the split sample-major copy, one 8 KB plane image (T | H | R | A) per 64-sample column
tile and k256 step, in the shared-memory layout of the wgmma B operand (geno_tile.cuh); the kernel only copies it.
Tiles (rt, ct) and (rt + 1, ct), row tiles counted from the job's first, run as one cluster that multicasts the plane
images; the rest (the second row's last column tiles, an odd last row tile) run in a second launch without a
partner.  The counts are checked against the oracle and the popcount kernel for even, odd and single row-tile
counts, a row block that starts on an odd row tile, the mapped (required-sample) job, and a seven-slot ring that
wraps twice and ends on a full or a short stage."""
import numpy as np
import pytest

from plink_ng_b200.host import KING_ALGO_POPCOUNT, KING_ALGO_TENSOR_TS, KingJob, MappedKingJob, pack_genotypes
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu


def _random_geno(m, n, seed, miss=0.05):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.02, 0.98, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _planes_numpy(geno):
    # [col tile][k256 step][plane][8-sample group][core matrix h][sample % 8][128 variant bits, little-endian]
    m, n = geno.shape
    n_pad, m_pad = -(-n // 640) * 640, -(-m // 256) * 256
    codes = np.full((n_pad, m_pad), 3, dtype=np.uint8)
    codes[:n, :m] = geno.T
    lo, hi = (codes & 1).astype(bool), (codes >> 1).astype(bool)
    pl = np.stack([lo & ~hi, ~lo, ~(lo | hi), ~lo & hi])  # [4][n_pad][m_pad]
    pl = pl.reshape(4, n_pad // 64, 8, 8, m_pad // 256, 2, 128).transpose(1, 4, 0, 2, 5, 3, 6)
    return np.packbits(pl, axis=-1, bitorder="little").reshape(-1)


def _counts(ctx, geno, r0=0, r1=None, algo=KING_ALGO_TENSOR_TS, max_variants_per_add=0):
    n = geno.shape[1]
    with KingJob(ctx, n, r0, n if r1 is None else r1, algo, max_variants_per_add) as job:
        job.add_variants(pack_genotypes(geno))
        return job.counts()


# the last k256 step short (300 and 1,000 variants), padding samples (136, 700) and more than one column tile
@pytest.mark.parametrize("m,n", [(300, 136), (1000, 700), (512, 64)])
def test_plane_copy_matches_numpy(gpu_ctx, m, n):
    geno = _random_geno(m, n, seed=m + n)
    want = _planes_numpy(geno)
    with KingJob(gpu_ctx, n, 0, n, KING_ALGO_TENSOR_TS) as job:
        job.add_variants(pack_genotypes(geno))
        got = job.last_planes(want.size)
    assert np.array_equal(got, want)


# 1 row tile (no pair), 2 (one pair row, lone edge tiles), 3 (odd: a last row tile alone), 4 and 5 row tiles
@pytest.mark.parametrize("n", [100, 200, 300, 500, 600])
def test_row_tile_counts_match_oracle_and_popcount(gpu_ctx, n):
    geno = _random_geno(1300, n, seed=n)
    got = _counts(gpu_ctx, geno)
    assert np.array_equal(got, orc.king_counts(geno))
    assert np.array_equal(got, _counts(gpu_ctx, geno, algo=KING_ALGO_POPCOUNT))


# a row block that starts on an odd row tile (row_start 128: pairs are row tiles 1 + 2, 3 + 4, ...), or inside one
@pytest.mark.parametrize("r0,r1", [(128, 600), (128, 520), (128, 256), (200, 600)])
def test_row_block_from_odd_tile(gpu_ctx, r0, r1):
    n = 600
    geno = _random_geno(900, n, seed=r0 + r1)
    got = _counts(gpu_ctx, geno, r0, r1)
    assert np.array_equal(got, orc.king_counts(geno, r0, r1))
    assert np.array_equal(got, _counts(gpu_ctx, geno, r0, r1, algo=KING_ALGO_POPCOUNT))


# seven slots of two k256 steps (3,584 variants): 29 steps (7,200 padded; the last stage short), 30, 31 and 32
@pytest.mark.parametrize("m", [7200, 7680, 7936, 8192])
def test_ring_wraps_twice_and_ends_full_or_short(gpu_ctx, m):
    geno = _random_geno(m, 200, seed=m)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


def test_launches_reuse_both_plane_copies(gpu_ctx):
    geno = _random_geno(5000, 300, seed=5)
    n = geno.shape[1]
    with KingJob(gpu_ctx, n, 0, n, KING_ALGO_TENSOR_TS, 1024) as job:
        for part in np.split(geno, [900, 2048, 2100, 3500]):
            job.add_variants(pack_genotypes(part))
        got = job.counts()
    assert np.array_equal(got, orc.king_counts(geno))


@pytest.mark.parametrize("xor", [False, True])
def test_mapped_job_with_required_samples(gpu_ctx, xor):
    n, m = 420, 3000
    geno = _random_geno(m, n, seed=420 + xor)
    rng = np.random.default_rng(4)
    mask = np.zeros(n, dtype=bool)
    mask[rng.choice(n, size=150, replace=False)] = True
    order = np.concatenate([np.flatnonzero(~mask), np.flatnonzero(mask)]).astype(np.uint32)
    n0 = n - int(mask.sum())
    col_end = n0 if xor else n
    with MappedKingJob(gpu_ctx, n, order, n0, n, col_end, max_variants_per_add=4096) as job:
        job.add_variants(pack_genotypes(geno))
        got = job.counts()
    full = orc.king_counts(geno[:, order], n0, n)
    keep = np.concatenate([np.arange(j) < col_end for j in range(n0, n)])
    assert np.array_equal(got, full[keep])
