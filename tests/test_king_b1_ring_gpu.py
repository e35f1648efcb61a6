"""GPU: the default KING kernel's operand ring and row-word look-ahead, bit-exact against the oracle.

The consumers load the row words of the next k256 step while the current step's wgmma group is issued, and the
first step of a stage only after that stage's slot is full; the slot goes back to the copier once its last group
has retired.  The sample-major copy keeps each sample's k256 step as one 64-byte piece with the k32 words in the
order 0, 4, 1, 5, 2, 6, 3, 7.  These cases wrap the five-slot ring (2,560 variants) at least twice and end on a full
or a short stage, put codes on one k32 word of every step at a time, span more than one row and column tile, reuse
both staged blocks over many launches, and run the mapped (required-sample) job on the same kernel."""
import numpy as np
import pytest

from plink_ng_b200.host import KING_ALGO_TENSOR_TS, KingJob, MappedKingJob, pack_genotypes
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu


def _random_geno(m, n, seed, miss=0.03):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.02, 0.98, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _structured(m, n):
    # every pair of codes meets at every variant position; the pattern moves with the bit position and the k32 step
    v = np.arange(m, dtype=np.int64)[:, None]
    s = np.arange(n, dtype=np.int64)[None, :]
    blk = s // 4
    return ((s + blk * (v % 32) + (blk * blk + 1) * (v // 32)) % 4).astype(np.uint8)


def _counts(ctx, geno, max_variants_per_add=0, pieces=None):
    n = geno.shape[1]
    with KingJob(ctx, n, 0, n, KING_ALGO_TENSOR_TS, max_variants_per_add) as job:
        for part in np.split(geno, np.cumsum(pieces)[:-1], axis=0) if pieces else [geno]:
            job.add_variants(pack_genotypes(part))
        return job.counts()


# 24 and 25 k256 steps: 12 full stages, or 12 and a short one; 5,890 and 6,300 are padded to them
@pytest.mark.parametrize("m", [5890, 6144, 6300, 6400])
@pytest.mark.parametrize("n", [136, 200])
def test_ring_wraps_twice_and_ends_full_or_short(gpu_ctx, m, n):
    geno = _random_geno(m, n, seed=m * 7 + n)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


# only the variants of k32 word k32 of each k256 step keep their codes, over 11 steps (6 stages, the last short)
@pytest.mark.parametrize("k32", range(8))
def test_each_k32_word_over_several_stages(gpu_ctx, k32):
    m = 11 * 256
    geno = _structured(m, 136)
    geno[(np.arange(m) % 256) // 32 != k32] = 3
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


def test_uneven_pieces_reuse_both_staged_blocks(gpu_ctx):
    # 1,024-variant batches: every add ends on a partial batch, so consecutive launches alternate the two blocks with
    # different variant counts (short stages included)
    geno = _random_geno(7000, 200, seed=77)
    pieces = [700, 1500, 37, 2048, 900, 1815]
    assert sum(pieces) == geno.shape[0]
    assert np.array_equal(_counts(gpu_ctx, geno, max_variants_per_add=1024, pieces=pieces), orc.king_counts(geno))


@pytest.mark.parametrize("xor", [False, True])
def test_mapped_job_with_required_samples(gpu_ctx, xor):
    n, m = 200, 6000
    geno = _random_geno(m, n, seed=6000 + xor)
    rng = np.random.default_rng(3)
    mask = np.zeros(n, dtype=bool)
    mask[rng.choice(n, size=70, replace=False)] = True
    order = np.concatenate([np.flatnonzero(~mask), np.flatnonzero(mask)]).astype(np.uint32)
    n0 = n - int(mask.sum())
    col_end = n0 if xor else n
    with MappedKingJob(gpu_ctx, n, order, n0, n, col_end, max_variants_per_add=4096) as job:
        job.add_variants(pack_genotypes(geno))
        got = job.counts()
    full = orc.king_counts(geno[:, order], n0, n)
    keep = np.concatenate([np.arange(j) < col_end for j in range(n0, n)])
    assert np.array_equal(got, full[keep])
