"""GPU parity: genotype counts, r^2 decision band and the full --indep-pairwise keep-list vs the
oracle (bit-exact) and vs the reference binary's own .prune.in files."""
import os

import numpy as np
import pytest

from plink_ng_b200.host import geno_counts, indep_pairwise, ld_band_flags, pack_genotypes
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu


def _ld_geno(m, n, seed, miss=0.02, ld=0.6):
    """Haplotype-copy model so neighbouring variants are in LD (as the reference's --dummy does)."""
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.03, 0.97, size=m)
    h = np.zeros((2, m, n), dtype=np.uint8)
    for k in range(2):
        cur = (rng.random(n) < freq[0]).astype(np.uint8)
        h[k, 0] = cur
        for v in range(1, m):
            fresh = (rng.random(n) < freq[v]).astype(np.uint8)
            copy = rng.random(n) < ld
            cur = np.where(copy & (rng.random() < 0.7), cur, fresh)
            h[k, v] = cur
    g = (h[0] + h[1]).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    g[5] = 0  # monomorphic
    g[6] = 1  # all het
    g[7] = 3  # all missing
    return g


def test_geno_counts(gpu_ctx):
    g = _ld_geno(700, 333, seed=1)
    got = geno_counts(gpu_ctx, pack_genotypes(g), 333)
    want = np.stack(orc.genotype_counts(g), axis=1)
    assert np.array_equal(got.astype(np.int64), want)


_FOUNDER_EDGES = [(n, 300, 70) for n in (1, 2, 31, 32, 33, 63, 65, 127, 129)]  # 64-founder stages
_BAND_EDGES = [(150, 700, band) for band in (1, 2, 63, 64, 65, 127, 128, 129)] + [(150, 120, 200)]  # column tiles of 64; band > m


@pytest.mark.parametrize("n,m,band", [(64, 200, 17), (333, 700, 49), (1000, 300, 130), (2100, 900, 500)] + _FOUNDER_EDGES + _BAND_EDGES)
def test_ld_band_flags_match_oracle(gpu_ctx, n, m, band):
    """The pair kernel (int8 tensor contraction over the founders, ld_ts_kernel.cuh) against the oracle's exact
    integer sums and fp64 test, pair by pair (only pairs with b >= 0: the other entries of a row are never written)."""
    g = _ld_geno(m, n, seed=n + m)
    thr = 0.2 * (1 + orc.SMALL_EPSILON)
    got = ld_band_flags(gpu_ctx, pack_genotypes(g), n, band, thr)
    x = np.where(g == 0, 1.0, np.where(g == 2, -1.0, 0.0)).astype(np.float32)
    nm = (g != 3).astype(np.float32)
    for a in range(1, m):
        bs = np.arange(max(0, a - band), a)
        nm_ct, s_b, q_b, s_a, q_a, dot = orc.ld_pair_components(x, nm, a, bs)
        cov12 = (dot * nm_ct - s_b * s_a).astype(np.float64)
        var1 = (q_b * nm_ct - s_b * s_b).astype(np.float64)
        var2 = (q_a * nm_ct - s_a * s_a).astype(np.float64)
        want = cov12 * cov12 > thr * var1 * var2
        assert np.array_equal(got[a, a - bs - 1].astype(bool), want), a


@pytest.mark.parametrize("window,step,r2,is_bp", [(50, 5, 0.2, False), (30, 1, 0.5, False), (500, 50, 0.1, False), (3000, 1, 0.3, True)])
def test_indep_pairwise_matches_oracle(gpu_ctx, window, step, r2, is_bp):
    n, m = 220, 1500
    g = _ld_geno(m, n, seed=window)
    rng = np.random.default_rng(9)
    chrom = np.repeat(np.array([1, 2, 0, 3, 4], dtype=np.uint32), [600, 1, 99, 500, 300])  # singleton chr 2, unplaced block
    bps = np.cumsum(rng.integers(1, 400, size=m)).astype(np.uint32)
    bps[700:] += 100000  # a gap
    got = indep_pairwise(gpu_ctx, pack_genotypes(g), n, chrom, bps, window, step, r2, window_is_bp=is_bp)
    want = orc.ld_prune(g, chrom, bps.astype(np.int64), window, step, r2, window_is_bp=is_bp)
    placed = chrom != 0
    assert (got[~placed] == 2).all()
    assert np.array_equal(got[placed] == 1, want[placed])
    assert 0 < want.sum() < m


def test_indep_pairwise_golden_reference_lists(gpu_ctx, golden_dir):
    geno = orc.read_bed(os.path.join(golden_dir, "a.bed"), 100)
    chrom, ids, bps = orc.read_bim(os.path.join(golden_dir, "a.bim"))
    codes = np.array([int(c) for c in chrom], dtype=np.uint32)
    gv = pack_genotypes(geno)
    for fname, window, step, r2, is_bp in (("a_ld.prune.in", 50, 5, 0.2, False), ("a_ld2.prune.in", 100, 1, 0.1, False), ("a_ldkb.prune.in", 20000, 1, 0.3, True)):
        removed = indep_pairwise(gpu_ctx, gv, 100, codes, bps, window, step, r2, window_is_bp=is_bp)
        kept = [ids[k] for k in range(len(ids)) if removed[k] == 0]
        ref = [ln.strip() for ln in open(os.path.join(golden_dir, fname)) if ln.strip()]
        assert kept == ref, fname
