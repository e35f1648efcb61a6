"""GPU: the split {lo32, hi32} form of the sample-major copy that the default KING kernel reads (geno_tile.cuh).
Structured genotypes put every pair of codes (i, j) on every bit position of a 32-variant word and on every k32
offset of a k256 step, bit-exact against the oracle.  The per-offset cases keep one variant position of the k256
step and make every other one missing, so a wrong bit mapping fails the case of the offset it breaks and names
the bit position."""
import numpy as np
import pytest

from plink_ng_b200.host import KING_ALGO_TENSOR_TS, KingJob, pack_genotypes
from oracle import plink_oracle as orc


def _structured(m, n):
    # samples in blocks of four: within a block the four codes are a rotation, so every variant holds every code
    # n / 4 times and every pair of codes (i, j) meets at every variant position; the rotation of each block moves
    # with the bit position (v % 32) and the k32 step (v // 32) at its own rate, so pairs of samples see different
    # code pairs from one position to the next
    v = np.arange(m, dtype=np.int64)[:, None]
    s = np.arange(n, dtype=np.int64)[None, :]
    blk = s // 4
    return ((s + blk * (v % 32) + (blk * blk + 1) * (v // 32)) % 4).astype(np.uint8)


def _counts(ctx, geno):
    n = geno.shape[1]
    with KingJob(ctx, n, 0, n, KING_ALGO_TENSOR_TS) as job:
        job.add_variants(pack_genotypes(geno))
        return job.counts()


def test_structured_codes_cover_every_pair_at_every_position():
    g = _structured(256, 16)
    for p in range(256):
        pairs = {(int(a), int(b)) for a in g[p] for b in g[p]}
        assert len(pairs) == 16, p


# 32 k +- 1 variants: words cut one variant short of or past a word boundary, inside and at the end of k256 steps
# and stages (a stage is two k256 steps); 136 samples span two row tiles and three column tiles
@pytest.mark.gpu
@pytest.mark.parametrize("m", [31, 33, 223, 225, 255, 257, 287, 289, 511, 513])
def test_structured_codes_match_oracle(gpu_ctx, m):
    geno = _structured(m, 136)
    assert np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno))


@pytest.mark.gpu
@pytest.mark.parametrize("k32", range(8))
def test_each_bit_position_alone_matches_oracle(gpu_ctx, k32):
    # 512 variants = one stage of two k256 steps; only variants at position 32 k32 + b of each step keep their codes
    base = _structured(512, 72)
    wrong = []
    for b in range(32):
        geno = base.copy()
        geno[np.arange(512) % 256 != 32 * k32 + b] = 3
        if not np.array_equal(_counts(gpu_ctx, geno), orc.king_counts(geno)):
            wrong.append(b)
    assert not wrong, f"k32 offset {k32}: counts differ from the oracle at bit positions {wrong}"
