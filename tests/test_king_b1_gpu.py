"""GPU: the default KING kernel on the binary tensor pipe (AND-POPC wgmma on T | H | R | A bit planes, stages of
two k256 steps, a short last stage when the block holds an odd number of 256-variant steps) at the variant counts,
genotype patterns, tile edges, row pieces and batch splits where its planes, stages or SS = HH - 2 IBS0 epilogue
could go wrong, bit-exact against the oracle or the popcount kernel."""
import numpy as np
import pytest

from plink_ng_b200.host import KING_ALGO_POPCOUNT, KING_ALGO_TENSOR_TS, KingJob, pack_genotypes, parallel_bounds
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu


def _random_geno(m, n, seed, miss=0.03):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.02, 0.98, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _counts(ctx, geno, algo=KING_ALGO_TENSOR_TS, r0=0, r1=None, max_variants_per_add=0, pieces=1):
    n = geno.shape[1]
    with KingJob(ctx, n, r0, n if r1 is None else r1, algo, max_variants_per_add) as job:
        for part in np.array_split(geno, pieces, axis=0):
            job.add_variants(pack_genotypes(part))
        return job.counts()


def test_selftest_b1_layout(gpu_ctx):
    # int8 and binary wgmma forms against host references; the binary case fixes the K-bit order of A and B
    gpu_ctx.selftest_umma(verbose=True)


# A stage is 512 variants (two k256 steps) and the block is padded to 256: one short stage (1, 255, 256), one full
# stage (257, 511, 512), a full stage and a short one (513), and the benchmark's 131,072-variant batch.
@pytest.mark.parametrize("m", [1, 255, 256, 257, 511, 512, 513])
def test_variant_counts_match_oracle(gpu_ctx, m):
    geno = _random_geno(m, 150, seed=m + 11)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


def test_full_batch_matches_popcount(gpu_ctx):
    n, m = 130, 131072
    geno = _random_geno(m, n, seed=130131)
    want = _counts(gpu_ctx, geno, KING_ALGO_POPCOUNT, max_variants_per_add=m)
    assert np.array_equal(_counts(gpu_ctx, geno, max_variants_per_add=m), want)


def test_degenerate_columns_and_variants_match_oracle(gpu_ctx):
    # a sample missing at every variant, a variant missing in every sample, an all-het and an all-hom-ALT sample,
    # an all-hom-REF sample, and two all-het / all-hom-ALT variants
    n, m = 200, 777
    geno = _random_geno(m, n, seed=2024)
    geno[:, 5] = 3
    geno[:, 64] = 1
    geno[:, 127] = 2
    geno[:, 128] = 0
    geno[300, :] = 3
    geno[301, :] = 1
    geno[513, :] = 2
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


# 128-row tile edges (127, 128, 129, 255, 257) and 64-column ones (191, 192)
@pytest.mark.parametrize("n", [127, 128, 129, 191, 192, 255, 257])
def test_tile_edges_match_oracle(gpu_ctx, n):
    geno = _random_geno(600, n, seed=n + 3)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


def test_parallel_bounds_row_pieces_match_oracle(gpu_ctx):
    n = 400
    geno = _random_geno(900, n, seed=4009)
    want = orc.king_counts(geno)
    tri = lambda r: r * (r - 1) // 2  # noqa: E731
    for piece in range(3):
        r0, r1 = parallel_bounds(n, 1, piece, 3)
        assert np.array_equal(_counts(gpu_ctx, geno, r0=r0, r1=r1), want[tri(r0) : tri(r1)])


def test_forced_multi_pass_matches_oracle(gpu_ctx):
    # 256-variant batches (one short stage each) over three adds: the raw accumulators, SS included, add up across
    # kernel launches
    geno = _random_geno(1800, 170, seed=1700)
    assert np.array_equal(_counts(gpu_ctx, geno, max_variants_per_add=256, pieces=3), orc.king_counts(geno))
