"""GPU: the default KING kernel's reduction epilogue.

Every CTA adds its tile's counts to the raw accumulators with `red.global.add`, row-tile pairs (2-CTA clusters) and
tiles without a partner alike.  The raw counts are compared exactly with the numpy oracle and the popcount kernel at
odd and even row-tile counts and column counts, row blocks from odd and even row tiles, mapped jobs whose column bound
cuts the triangle, short last stages and rings that wrap twice, and several batches into one job (the reductions of
every launch add up)."""
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


def _counts(ctx, geno, r0=0, r1=None, algo=KING_ALGO_TENSOR_TS, max_variants_per_add=0):
    n = geno.shape[1]
    with KingJob(ctx, n, r0, n if r1 is None else r1, algo, max_variants_per_add) as job:
        job.add_variants(pack_genotypes(geno))
        return job.counts()


# 1 row tile (no pair), 3 (a last row tile alone), 5 (alone, with 9 column tiles), 6 (the second row of the last pair
# with one column tile more than the first) and 8 row tiles
@pytest.mark.parametrize("n", [100, 300, 520, 700, 1000])
def test_counts_match_oracle_and_popcount(gpu_ctx, n):
    geno = _random_geno(1300, n, seed=n)
    got = _counts(gpu_ctx, geno)
    assert np.array_equal(got, orc.king_counts(geno))
    assert np.array_equal(got, _counts(gpu_ctx, geno, algo=KING_ALGO_POPCOUNT))


# row blocks from an odd row tile (128: pairs are row tiles 1 + 2, 3 + 4, ...), an even one (256), and inside a tile
@pytest.mark.parametrize("r0,r1", [(128, 700), (256, 700), (256, 520), (200, 1000), (384, 512)])
def test_row_blocks_from_odd_and_even_tiles(gpu_ctx, r0, r1):
    n = r1 if r1 > 700 else 700
    geno = _random_geno(900, n, seed=r0 + r1)
    got = _counts(gpu_ctx, geno, r0, r1)
    assert np.array_equal(got, orc.king_counts(geno, r0, r1))
    assert np.array_equal(got, _counts(gpu_ctx, geno, r0, r1, algo=KING_ALGO_POPCOUNT))


@pytest.mark.parametrize("xor", [False, True])
def test_mapped_job_with_required_samples(gpu_ctx, xor):
    n, m = 700, 2000
    geno = _random_geno(m, n, seed=700 + xor)
    rng = np.random.default_rng(7)
    mask = np.zeros(n, dtype=bool)
    mask[rng.choice(n, size=280, replace=False)] = True  # rows 420-699; with xor, 7 column tiles
    order = np.concatenate([np.flatnonzero(~mask), np.flatnonzero(mask)]).astype(np.uint32)
    n0 = n - int(mask.sum())
    col_end = n0 if xor else n
    with MappedKingJob(gpu_ctx, n, order, n0, n, col_end, max_variants_per_add=4096) as job:
        job.add_variants(pack_genotypes(geno))
        got = job.counts()
    full = orc.king_counts(geno[:, order], n0, n)
    keep = np.concatenate([np.arange(j) < col_end for j in range(n0, n)])
    assert np.array_equal(got, full[keep])


# seven slots of two k256 steps: 29 steps (the last stage short), 31, and 32 (the ring wraps twice, ends full)
@pytest.mark.parametrize("m", [7200, 7936, 8192])
def test_short_last_stage_and_ring_wraps(gpu_ctx, m):
    geno = _random_geno(m, 520, seed=m)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


def test_batches_accumulate(gpu_ctx):
    geno = _random_geno(5000, 700, seed=11)
    n = geno.shape[1]
    with KingJob(gpu_ctx, n, 0, n, KING_ALGO_TENSOR_TS, 1024) as job:
        for part in np.split(geno, [700, 2048, 2100, 3500]):
            job.add_variants(pack_genotypes(part))
        got = job.counts()
    assert np.array_equal(got, orc.king_counts(geno))
