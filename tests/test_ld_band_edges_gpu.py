"""LD pair decisions (ld_ts_kernel through pl2gpu_ld_band_flags) at chunk edges, on rounding boundaries and at large
founder counts, every in-band pair against the reference's test restated in numpy.

The reference decides a pair (second = a, first = b = a - d) with cov12^2 > (t * var1) * var2 on the exact integer
sums over the founders, int64 -> double and unfused products in that order (plink2_ld.cc:1085-1090).  The oracle here
forms the six sums one diagonal offset d at a time, for all pairs (a, a - d) at once, and is itself checked against
orc.ld_pair_components.  Row a of the flag array holds flags[a * band + (d - 1)]; offsets d > a (pairs with b < 0) are
never written by the device and are never read here."""
from fractions import Fraction

import numpy as np
import pytest

from plink_ng_b200.host import ld_band_flags, pack_genotypes
from oracle import plink_oracle as orc

CHUNK = 16384  # kLdChunkVariants: variants per kernel launch of pl2gpu_ld_band_flags
THR = 0.2 * (1 + orc.SMALL_EPSILON)


def band_sums(geno, band):
    """(nm12, s_b, q_b, s_a, q_a, dot) [m, band] int64 of ComputeIndepPairwiseR2Components (plink2_ld.cc:699-723) for
    every pair (a, a - d), column d - 1; zero where a - d < 0."""
    x = np.where(geno == 0, 1, np.where(geno == 2, -1, 0)).astype(np.int8)
    nm = (geno != 3).astype(np.int8)
    hom = x * x
    m = geno.shape[0]
    out = np.zeros((6, m, band), dtype=np.int64)
    for d in range(1, min(band, m - 1) + 1):
        xa, na, ha, xb, nb, hb = x[d:], nm[d:], hom[d:], x[:-d], nm[:-d], hom[:-d]
        for k, (p, q) in enumerate(((na, nb), (xb, na), (hb, na), (xa, nb), (ha, nb), (xa, xb))):
            out[k, d:, d - 1] = (p * q).sum(axis=1, dtype=np.int64)
    return out


def pair_terms(sums):
    """cov12, var1, var2 as the doubles the reference compares."""
    nm12, s_b, q_b, s_a, q_a, dot = sums
    return (dot * nm12 - s_b * s_a).astype(np.float64), (q_b * nm12 - s_b * s_b).astype(np.float64), (q_a * nm12 - s_a * s_a).astype(np.float64)


def defined(m, band):
    """[m, band] mask of the pairs with b >= 0."""
    return np.arange(m)[:, None] >= np.arange(1, band + 1)[None, :]


def check_flags(got, terms, thr):
    cov, var1, var2 = terms
    want = cov * cov > thr * var1 * var2
    ok = defined(*got.shape)
    bad = np.argwhere(ok & (got.astype(bool) != want))
    assert bad.size == 0, f"{len(bad)} pair decisions differ at t = {thr!r}, first (a, d) = ({bad[0][0]}, {bad[0][1] + 1})"
    return int(want[ok].sum())


def ld_geno(m, n, seed, miss=0.02, copy=0.6, lo=0.03):
    """Haplotype-copy model: neighbouring variants in LD; a few monomorphic / all-het / all-missing rows."""
    rng = np.random.default_rng(seed)
    freq = rng.uniform(lo, 1 - lo, size=m)
    fresh = rng.random((2, m, n)) < freq[None, :, None]
    keep = (rng.random((2, m, n)) < copy) & (rng.random((2, m, 1)) < 0.7)
    h = fresh.copy()
    for v in range(1, m):
        h[:, v] = np.where(keep[:, v], h[:, v - 1], fresh[:, v])
    g = (h[0].astype(np.uint8) + h[1]).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    if m > 40:
        g[5], g[6], g[7] = 0, 1, 3
    return g


def test_band_sums_match_pair_components():
    g = ld_geno(150, 70, seed=3)
    band = 40
    sums = band_sums(g, band)
    x = np.where(g == 0, 1.0, np.where(g == 2, -1.0, 0.0)).astype(np.float32)
    nm = (g != 3).astype(np.float32)
    for a in range(1, 150):
        bs = np.arange(max(0, a - band), a)
        want = np.stack(orc.ld_pair_components(x, nm, a, bs))
        assert np.array_equal(sums[:, a, a - bs - 1], want), a
    assert not sums[:, 0].any() and not sums[:, 3, 3:].any()


# ------------------------------------------------------------------------------------------------------- device
@pytest.mark.gpu
@pytest.mark.parametrize("m,band,n", [(CHUNK + 1, 1, 40), (CHUNK + 1, 64, 96), (CHUNK + 700, 65, 40), (CHUNK + 700, 500, 96), (2 * CHUNK + 65, 130, 40), (2 * CHUNK + 65, 65, 96)])
def test_ld_chunk_edges(gpu_ctx, m, band, n):
    """A second chunk re-stages roundup(band, 64) rows of the first; 2 x 16,384 + 65 variants run three chunks, so both
    flag buffers are drained and reused."""
    g = ld_geno(m, n, seed=m + band + n)
    got = ld_band_flags(gpu_ctx, pack_genotypes(g), n, band, THR)
    flagged = check_flags(got, pair_terms(band_sums(g, band)), THR)
    assert 0 < flagged < defined(m, band).sum()


def _exact_over(c, v1, v2, thr):
    return Fraction(int(c)) ** 2 > Fraction(thr) * int(v1) * int(v2)


def _tie_thresholds(terms, want_ct=3):
    """Thresholds equal to the fp64 r^2 of pairs (or one ulp away) where the reference's rounded test decides the pair
    differently from t * (var1 * var2), or from the exact comparison (what a fused or reordered product computes)."""
    cov, var1, var2 = (t.ravel() for t in terms)
    live = np.flatnonzero(var1 * var2 > 0)
    c2, p1, p2 = cov[live] ** 2, var1[live], var2[live]
    r2 = c2 / (p1 * p2)
    reorder, exact = [], []
    for cand in (r2, np.nextafter(r2, 0), np.nextafter(r2, 2)):
        ref = c2 > cand * p1 * p2
        for k in np.flatnonzero(ref != (c2 > cand * (p1 * p2)))[:want_ct]:
            reorder.append(float(cand[k]))
        near = np.flatnonzero(np.abs(c2 - cand * p1 * p2) <= 1e-13 * c2)
        for k in near[:400]:
            if len(exact) < want_ct and bool(ref[k]) != _exact_over(cov[live[k]], p1[k], p2[k], float(cand[k])):
                exact.append(float(cand[k]))
    return reorder[:want_ct], exact


def _repeat_block(base, reps):
    """`base` repeated, alleles flipped (0 <-> 2) in every other copy: many pairs share their sums, and pairs of a
    variant with its copies have r^2 = 1."""
    flip = np.where(base == 3, 3, 2 - np.minimum(base, 2)).astype(np.uint8)
    return np.concatenate([flip if r & 1 else base for r in range(reps)])


@pytest.mark.gpu
def test_ld_decisions_on_rounding_boundaries(gpu_ctx):
    n, band = 300, 70
    g = _repeat_block(ld_geno(37, n, seed=17, copy=0.8, lo=0.15), 16)
    m = g.shape[0]
    terms = pair_terms(band_sums(g, band))
    cov, var1, var2 = terms
    ok = defined(m, band)
    dup = ok & (var1 > 0) & (cov * cov == var1 * var2)
    assert dup.sum() >= 500  # a variant and its copies, flipped or not
    reorder, exact = _tie_thresholds(terms)
    assert reorder and exact, (reorder, exact)
    with np.errstate(invalid="ignore"):
        r2 = (cov * cov) / (var1 * var2)
    chosen = [float(r2[a, d - 1]) for a, d in ((300, 2), (301, 10), (450, 33), (500, 60))]
    for thr in chosen:  # pairs with the same sums as the one that set the threshold sit on the same boundary
        assert (ok & (r2 == thr)).sum() >= 8, thr
    gv = pack_genotypes(g)
    for thr in reorder + exact + chosen + [t * (1 + orc.SMALL_EPSILON) for t in chosen] + [1.0, 1 - 2.0**-40]:
        got = ld_band_flags(gpu_ctx, gv, n, band, thr)
        check_flags(got, terms, thr)
        if thr == 1.0:
            assert not got[dup].any()
        elif thr == 1 - 2.0**-40:
            assert got[dup].all()


@pytest.mark.gpu
def test_ld_large_founder_counts(gpu_ctx):
    """16,000 founders, strongly linked neighbours near frequency 1/2: cov^2 passes 2^53 and is rounded before the
    comparison, as in the reference."""
    n, m, band = 16000, 400, 65
    g = ld_geno(m, n, seed=23, miss=0.01, copy=0.97, lo=0.4)
    g[100] = g[99]
    g[200] = np.where(g[199] == 3, 3, 2 - np.minimum(g[199], 2))
    terms = pair_terms(band_sums(g, band))
    cov = terms[0]
    ok = defined(m, band)
    assert (ok & (cov * cov > 2.0**53)).sum() > 10
    reorder, exact = _tie_thresholds(terms, want_ct=2)
    gv = pack_genotypes(g)
    for thr in [THR, 0.9] + reorder + exact:
        got = ld_band_flags(gpu_ctx, gv, n, band, thr)
        check_flags(got, terms, thr)
