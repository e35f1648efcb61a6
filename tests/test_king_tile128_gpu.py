"""GPU: the default KING kernel (one CTA per 128 x 64 pair tile, bulk-copied raw words, 3-stage ring of 256
variants) at the variant counts, sample counts and row ranges where its ring, tile edges or 64-column read-backs
could go wrong, bit-exact against the oracle or the popcount kernel."""
import numpy as np
import pytest

from plink_ng_b200.host import KING_ALGO_POPCOUNT, KING_ALGO_TENSOR, KING_ALGO_TENSOR_TS, KingJob, pack_genotypes, parallel_bounds
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu


def _random_geno(m, n, seed, miss=0.03):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.02, 0.98, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _counts(ctx, geno, algo=KING_ALGO_TENSOR_TS, r0=0, r1=None, max_variants_per_add=0):
    n = geno.shape[1]
    with KingJob(ctx, n, r0, n if r1 is None else r1, algo, max_variants_per_add) as job:
        job.add_variants(pack_genotypes(geno))
        return job.counts()


# Variants are padded to 256 and staged 256 at a time in a ring of 3: 1, 2, 3, 4 and 13 stages.
@pytest.mark.parametrize("m", [1, 300, 700, 1000, 3300])
def test_ring_stages_match_oracle(gpu_ctx, m):
    geno = _random_geno(m, 200, seed=m + 7)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


# Column tiles are 64 samples wide: one partial tile (2, 63), exactly one (64), one sample past it (65), a last
# column tile with one real sample (193 = 3 * 64 + 1), and 641 samples (padding to 640 + 640).
@pytest.mark.parametrize("n", [2, 63, 64, 65, 193, 641])
def test_column_tile_edges_match_oracle(gpu_ctx, n):
    geno = _random_geno(600, n, seed=n)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


def test_row_piece_inside_row_tile_matches_oracle(gpu_ctx):
    n = 641
    geno = _random_geno(800, n, seed=6410)
    want = orc.king_counts(geno)
    tri = lambda r: r * (r - 1) // 2  # noqa: E731
    for piece in range(4):
        r0, r1 = parallel_bounds(n, 1, piece, 4)  # (1, 321), (321, 454), (454, 556), (556, 641)
        assert r0 % 128 != 0
        assert np.array_equal(_counts(gpu_ctx, geno, r0=r0, r1=r1), want[tri(r0) : tri(r1)])


def test_full_batch_three_algorithms_agree(gpu_ctx):
    # one 131,072-variant add, the batch the benchmark times, at a sample count that ends in a one-sample column tile
    n, m = 193, 131072
    geno = _random_geno(m, n, seed=193131)
    res = [_counts(gpu_ctx, geno, algo, max_variants_per_add=m) for algo in (KING_ALGO_POPCOUNT, KING_ALGO_TENSOR, KING_ALGO_TENSOR_TS)]
    assert np.array_equal(res[0], res[1]) and np.array_equal(res[0], res[2])


def test_kinship_and_filtered_readbacks_equal_popcount(gpu_ctx):
    # 64-column finalize and filter kernels against the popcount job's 96-column ones; a few duplicated samples
    # give pairs above the filter threshold in several column tiles
    n = 321
    geno = _random_geno(2000, n, seed=321)
    for dst, src in ((70, 3), (200, 66), (320, 130), (129, 128)):
        geno[:, dst] = geno[:, src]
    out = {}
    for algo in (KING_ALGO_POPCOUNT, KING_ALGO_TENSOR_TS):
        with KingJob(gpu_ctx, n, 0, n, algo) as job:
            job.add_variants(pack_genotypes(geno))
            r0, r1 = 100, 300
            out[algo] = (job.kinship(), job.kinship(r0, r1), job.filtered(0.2), job.filtered(-0.05, row_start=r0, row_end=r1))
    want_kin = orc.king_kinship(orc.king_counts(geno))
    got, ref = out[KING_ALGO_TENSOR_TS], out[KING_ALGO_POPCOUNT]
    assert np.array_equal(got[0], want_kin, equal_nan=True)
    assert np.array_equal(got[1], ref[1], equal_nan=True)
    for g, r in ((got[2], ref[2]), (got[3], ref[3])):
        assert np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1]) and np.array_equal(g[2], r[2], equal_nan=True)
    assert len(got[2][0]) >= 4 and len(got[3][0]) > len(got[2][0])
