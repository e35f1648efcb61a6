"""GPU: the KING tensor kernels' shared-memory ring (producer warpgroup -> consumer warpgroups) at the variant
counts, tile edges and batch shape where its stage bookkeeping could go wrong, bit-exact against the oracle or
the popcount kernel."""
import numpy as np
import pytest

from plink_ng_b200.host import KING_ALGO_POPCOUNT, KING_ALGO_TENSOR, KING_ALGO_TENSOR_TS, KingJob, pack_genotypes, parallel_bounds
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu

ALGOS = [pytest.param(KING_ALGO_TENSOR, id="tensor"), pytest.param(KING_ALGO_TENSOR_TS, id="tensor_ts")]


def _random_geno(m, n, seed, miss=0.03):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.02, 0.98, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _counts(ctx, geno, algo, r0=0, r1=None, max_variants_per_add=0):
    n = geno.shape[1]
    with KingJob(ctx, n, r0, n if r1 is None else r1, algo, max_variants_per_add) as job:
        job.add_variants(pack_genotypes(geno))
        return job.counts()


# Variants are padded to 256.  The 80-column kernel stages 256 variants at a time in a ring of 3, the 96-column
# kernel 128 at a time in a ring of 4, so these counts give the 80-column ring 1, 1, 2, 3, 4 and 13 stages (one
# pass, a wrap, several odd wraps) and the 96-column ring 2, 2, 4, 6, 8 and 26.
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("m", [1, 200, 500, 700, 1000, 3300])
def test_ring_stage_counts_match_oracle(gpu_ctx, algo, m):
    geno = _random_geno(m, 150, seed=m)
    assert np.array_equal(_counts(gpu_ctx, geno, algo), orc.king_counts(geno))


# 641 samples: the 80-column kernel pads samples to 640, so the last column tile holds one real sample and 79
# padding columns.  The middle ParallelBounds piece starts at row 371, inside a 128-row tile.
@pytest.mark.parametrize("algo", ALGOS)
def test_tile_edges_match_oracle(gpu_ctx, algo):
    n, m = 641, 600
    geno = _random_geno(m, n, seed=641)
    want = orc.king_counts(geno)
    assert np.array_equal(_counts(gpu_ctx, geno, algo), want)
    r0, r1 = parallel_bounds(n, 1, 1, 3)
    assert r0 % 128 != 0
    tri = lambda r: r * (r - 1) // 2  # noqa: E731
    assert np.array_equal(_counts(gpu_ctx, geno, algo, r0, r1), want[tri(r0) : tri(r1)])


def test_full_batch_tensor_equals_popcount(gpu_ctx):
    # one 131,072-variant add, the batch the benchmark times, through a job sized for it
    n, m = 1000, 131072
    rng = np.random.default_rng(131072)
    geno = rng.integers(0, 4, size=(m, n), dtype=np.uint8)
    res = [_counts(gpu_ctx, geno, algo, max_variants_per_add=m) for algo in (KING_ALGO_POPCOUNT, KING_ALGO_TENSOR, KING_ALGO_TENSOR_TS)]
    assert np.array_equal(res[0], res[1]) and np.array_equal(res[0], res[2])
    assert res[0][:, 4].max() <= m and res[0][:, 4].min() > 0
