"""The two products of `--pca approx` (pca_ts_kernels.cuh through pl2gpu_pca_products) and `--variant-score` at their
tile, column-group, chunk and split-K edges against exact references, under the per-entry error bounds of DESIGN §4.

Y is the job's standardised matrix: y_vs = sl_v g_vs + ic_v m_vs (g the ALT dosage, missing 0; m the non-missing
indicator).  The dense operand is encoded per column c with a scale 2^F_c, F_c = 30 - e_c where
2^(e_c - 1) <= M_c = max |x| < 2^e_c (an all-zero column: F = 0): pass 0 carries q0 = rn(x 2^F), pass 1
q1 = rn((x 2^F - q0) 2^30), so the encoded operand is within 2^-(F_c + 31) <= M_c 2^-60 of x.  Every product of the
digits is exact integer arithmetic; what remains is that quantisation and the fp64 epilogues:

  XA   |dH_vc| <= 2^-(F_c+31) (|sl_v| sum_s g_vs + |ic_v| sum_s m_vs) + gamma_8 (|sl_v| sum_s g_vs |G_sc| + |ic_v| sum_s m_vs |G_sc|)
  XtB  |dO_sc| <= 2^-(F_c+31) sum_v (g_vs + m_vs) + gamma_(splits+4) sum_v (g_vs |sl_v H_vc| + m_vs |ic_v H_vc|)
       with F_c from max_v max(|sl_v H_vc|, |ic_v H_vc|): both planes share one scale
  vscore (slope 1, icpt -2f, plus 2f sum_s w_s):
       |dS_vc| <= 2^-(F_c+31) (sum_s g_vs + 2f_v sum_s m_vs) + gamma_(n+8) (sum_s g_vs |w_sc| + 2f_v sum_s |w_sc|)

gamma_k = k u / (1 - k u), u = 2^-53.  The references are exact up to one long-double rounding: the operand is split
exactly as x = q0 2^-F + q1 2^-(F+30) + r, the integer parts are contracted exactly and r (below 2^-(F+31)) in fp64;
the products sl_v H_vc enter as exact double-double pairs."""
import os
import subprocess

import numpy as np
import pytest

from oracle import plink_oracle as orc
from plink_ng_b200 import host
from plink_ng_b200.host import pack_genotypes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
ENV = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
LD = np.longdouble
UNIT = 2.0**-53
FIXED_BITS = 30  # kPcaFixedBits
PASS1_BITS = 30  # kPcaPass1Scale = 2^30
CG = 32  # kPcaCgMax: columns per launch
CHUNK = 65536  # pl2gpu_pca_add_variants uploads and standardises this many variants at a time
VSCORE_PIECE = 262144  # RunVscore: variants per job
# pca_xtb_wg_kernel's int32 digit accumulators gain at most 2 * 128 + 128 per variant, 32 variants per k-step
XTB_MAX_KSTEPS = (0x7FFFFFFF // (384 * 32)) // 4 * 4


def gamma(k):
    return k * UNIT / (1 - k * UNIT)


def col_scales(x):
    """F_c of every column of x (pca_scales_kernel)."""
    mx = np.abs(x).max(axis=0, initial=0.0)
    return np.where(mx > 0, FIXED_BITS - np.frexp(mx)[1], 0).astype(np.int64)


def encode(x, f, passes=2):
    """pca_digits_kernel's two passes restated: (q0, q1, r) with x = q0 2^-F + q1 2^-(F+30) + r exactly."""
    ys = np.ldexp(x, f[None, :])
    q0 = np.rint(ys)
    t = (ys - q0) * 2.0**PASS1_BITS
    q1 = np.rint(t) if passes == 2 else np.zeros_like(t)
    return q0, q1, np.ldexp(t - q1, -(f[None, :] + PASS1_BITS))


def exact_dot(a, x, f):
    """a @ x for small non-negative integers a [R, K] and fp64 x [K, C], in long double, exact up to its last rounding.
    The integer contractions run in fp64: every partial sum is an integer below 2^53."""
    a = np.asarray(a, dtype=np.float64)
    assert a.shape[1] * 2.0 * 2.0**31 < 2.0**53
    q0, q1, r = encode(x, f)
    return np.ldexp((a @ q0).astype(LD), -f) + np.ldexp((a @ q1).astype(LD), -(f + PASS1_BITS)) + (a @ r).astype(LD)


def two_prod(a, b):
    """(p, e) with a b = p + e exactly, p = fl(a b) (Dekker, no fused multiply-add needed)."""
    p = a * b

    def split(x):
        c = 134217729.0 * x
        hi = c - (c - x)
        return hi, x - hi

    ah, al = split(a)
    bh, bl = split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def planes(geno):
    return np.where(geno == 3, 0, geno).astype(np.float64), (geno != 3).astype(np.float64)


def filled_freqs(geno, ref_freq=None):
    own = orc.ref_allele_freqs(geno)
    return own if ref_freq is None else np.where(np.isnan(ref_freq), own, ref_freq)


def standardise(geno, ref_freq=None):
    """slope / intercept per variant as pl2gpu_pca_add_variants stores them for a PCA job."""
    rf = filled_freqs(geno, ref_freq)
    alt = 1.0 - rf
    var = 2 * rf * alt
    ok = var > orc.SMALL_EPSILON
    sl = np.where(ok, 1.0 / np.sqrt(np.where(ok, var, 1.0)), 0.0)
    return sl, np.where(ok, -2 * alt * sl, 0.0)


def xa_reference(geno, g, sl, ic):
    dos, nm = planes(geno)
    f = col_scales(g)
    return sl[:, None].astype(LD) * exact_dot(dos, g, f) + ic[:, None].astype(LD) * exact_dot(nm, g, f)


def xa_bound(geno, g, sl, ic):
    dos, nm = planes(geno)
    q = np.ldexp(1.0, -(col_scales(g) + FIXED_BITS + 1))[None, :]
    asl, aic = np.abs(sl)[:, None], np.abs(ic)[:, None]
    return q * (asl * dos.sum(1)[:, None] + aic * nm.sum(1)[:, None]) + gamma(8) * (asl * (dos @ np.abs(g)) + aic * (nm @ np.abs(g)))


def xtb_reference(geno, h, sl, ic):
    dos, nm = planes(geno)
    p1, e1 = two_prod(sl[:, None], h)
    p2, e2 = two_prod(ic[:, None], h)
    f = col_scales(np.concatenate([p1, p2]))
    return exact_dot(dos.T, p1, f) + exact_dot(nm.T, p2, f) + (dos.T @ e1 + nm.T @ e2).astype(LD)


def xtb_bound(geno, h, sl, ic, splits):
    dos, nm = planes(geno)
    p1, p2 = sl[:, None] * h, ic[:, None] * h
    q = np.ldexp(1.0, -(col_scales(np.concatenate([p1, p2])) + FIXED_BITS + 1))[None, :]
    return q * (dos.sum(0) + nm.sum(0))[:, None] + gamma(splits + 4) * (dos.T @ np.abs(p1) + nm.T @ np.abs(p2))


def _cdiv(a, b):
    return -(-a // b)


def xtb_plan(n, m, sms):
    """(splits, k-steps per split, k-steps) of Y^T H for a job announced with m variants (pca.cu, PcaTsAlloc)."""
    tiles2 = _cdiv(n, 128)
    ksteps = _cdiv(m, 128) * 128 // 32
    splits = max(1, min(_cdiv(2 * sms, tiles2), ksteps // 64))
    kps = min(XTB_MAX_KSTEPS, _cdiv(_cdiv(ksteps, splits), 4) * 4)
    return _cdiv(ksteps, kps), kps, ksteps


def vscore_reference(geno, w, rf):
    dos, nm = planes(geno)
    f = col_scales(w)
    tf = 2.0 * (1.0 - rf)
    return exact_dot(dos, w, f) + tf[:, None].astype(LD) * exact_dot(1.0 - nm, w, f)


def vscore_bound(geno, w, rf):
    dos, nm = planes(geno)
    tf = 2.0 * (1.0 - rf)
    q = np.ldexp(1.0, -(col_scales(w) + FIXED_BITS + 1))[None, :]
    aw = np.abs(w)
    return q * (dos.sum(1) + tf * nm.sum(1))[:, None] + gamma(w.shape[0] + 8) * (dos @ aw + tf[:, None] * aw.sum(0)[None, :])


def _check(got, want, bound, what):
    """Every entry within its bound; prints the largest error / bound ratio."""
    assert got.shape == want.shape == bound.shape, what
    err = np.abs(got.astype(LD) - want).astype(np.float64)
    bad = np.flatnonzero(~(err <= bound))
    assert bad.size == 0, f"{what}: {bad.size} of {err.size} entries outside the bound, e.g. {np.unravel_index(bad[0], err.shape)}: |err| {err.flat[bad[0]]:.3g} > {bound.flat[bad[0]]:.3g}"
    print(f"RATIO {what} {float((err / np.where(bound > 0, bound, np.inf)).max(initial=0.0)):.3g}")


def _geno(m, n, seed, miss=0.03, lo=0.02, mono_every=0):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(lo, 1 - lo, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    if mono_every:
        g[0::mono_every] = 0
        g[mono_every // 2 :: mono_every] = 2
    if miss:
        g[rng.random((m, n)) < miss] = 3
    return g


def _dense(rows, cols, seed):
    return np.random.default_rng(seed).standard_normal((rows, cols))


def _products(ctx, geno, g=None, h=None, ref_freq=None, calls=None, sms=None):
    """Both products of one job against their references; returns the XtB split count used by the bound."""
    m, n = geno.shape
    yg, yth = host.pca_products(ctx, pack_genotypes(geno), n, g, h, ref_freqs=ref_freq, calls=calls)
    sl, ic = standardise(geno, ref_freq)
    tag = f"n={n} m={m}"
    if g is not None:
        _check(yg, xa_reference(geno, g, sl, ic), xa_bound(geno, g, sl, ic), f"XA {tag} cx={g.shape[1]}")
    splits = None
    if h is not None:
        splits = xtb_plan(n, m, sms or _sm_count())[0]
        _check(yth, xtb_reference(geno, h, sl, ic), xtb_bound(geno, h, sl, ic, splits), f"XtB {tag} ct={h.shape[1]} splits={splits}")
    return splits


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------ the bounds themselves (CPU)
def _emulate_xa(geno, g, sl, ic, passes):
    """The device's XA arithmetic in numpy: exact digit sums, then its fp64 epilogue per pass."""
    dos, nm = planes(geno)
    f = col_scales(g)
    q0, q1, _ = encode(g, f, passes)
    inv = np.ldexp(1.0, -f)[None, :]
    h = (sl[:, None] * (dos @ q0) + ic[:, None] * (nm @ q0)) * inv
    if passes == 2:
        h = h + (sl[:, None] * (dos @ q1) + ic[:, None] * (nm @ q1)) * (inv * 2.0**-PASS1_BITS)
    return h


def _emulate_xtb(geno, h, sl, ic, splits, kps, passes):
    """The device's XtB arithmetic: per split exact digit sums -> fp64 partials, fixed-order reduce, pass 1 added."""
    dos, nm = planes(geno)
    p1, p2 = sl[:, None] * h, ic[:, None] * h
    f = col_scales(np.concatenate([p1, p2]))
    inv = np.ldexp(1.0, -f)[None, :]
    e1, e2 = encode(p1, f, passes), encode(p2, f, passes)
    out = np.zeros((geno.shape[1], h.shape[1]))
    for pas in range(passes):
        acc = np.zeros_like(out)
        for k in range(splits):
            s = slice(k * kps * 32, (k + 1) * kps * 32)
            acc = acc + (dos[s].T @ e1[pas][s] + nm[s].T @ e2[pas][s]) * inv
        out = out + acc * (2.0**-PASS1_BITS if pas else 1.0)
    return out


def test_bounds_hold_for_two_passes_and_catch_one():
    """The numpy restatement of the two-pass encoding stays inside both bounds; a single 30-bit pass exceeds them by
    orders of magnitude, so the bounds detect a lost pass."""
    geno = _geno(700, 90, seed=1, mono_every=17)
    sl, ic = standardise(geno)
    g = _dense(90, 5, 2) * np.array([1.0, 2.0**40, 2.0**-40, 0.0, 1.0])
    g[:, 3] = 0.0
    g[7, 4] = 1e9  # one dominant entry: the others keep fewer bits
    want, bound = xa_reference(geno, g, sl, ic), xa_bound(geno, g, sl, ic)
    err2 = np.abs(_emulate_xa(geno, g, sl, ic, 2).astype(LD) - want).astype(np.float64)
    assert np.all(err2 <= bound) and err2.max() > 0.0
    err1 = np.abs(_emulate_xa(geno, g, sl, ic, 1).astype(LD) - want).astype(np.float64)
    assert np.max(err1 / np.where(bound > 0, bound, np.inf)) > 1e6
    h = _dense(700, 4, 3) * np.array([1.0, 2.0**30, 2.0**-30, 1.0])
    h[5, 3] = 1e7
    splits, kps, _ = 3, 8, 22  # 22 k-steps (704 variants) in splits of 8, 8 and 6
    want, bound = xtb_reference(geno, h, sl, ic), xtb_bound(geno, h, sl, ic, splits)
    err2 = np.abs(_emulate_xtb(geno, h, sl, ic, splits, kps, 2).astype(LD) - want).astype(np.float64)
    assert np.all(err2 <= bound) and err2.max() > 0.0
    err1 = np.abs(_emulate_xtb(geno, h, sl, ic, splits, kps, 1).astype(LD) - want).astype(np.float64)
    assert np.max(err1 / bound) > 1e6


def test_exact_reference_is_exact():
    """exact_dot against Python's exact rational arithmetic on entries spanning 2^-60 .. 2^40 in one column."""
    from fractions import Fraction

    rng = np.random.default_rng(4)
    a = rng.integers(0, 3, size=(3, 50)).astype(np.float64)
    x = rng.standard_normal((50, 2)) * np.ldexp(1.0, rng.integers(-60, 40, size=(50, 1)))
    got = exact_dot(a, x, col_scales(x))
    for i in range(3):
        for c in range(2):
            exact = sum(Fraction(int(a[i, k])) * Fraction(float(x[k, c])) for k in range(50))
            assert abs(Fraction(*got[i, c].as_integer_ratio()) - exact) <= abs(exact) * Fraction(2.0**-61)


def test_xtb_plan_and_accumulator_cap():
    """The split plan restated from pca.cu, and the cap that keeps a split's int32 digit sums in range."""
    assert 384 * 32 * XTB_MAX_KSTEPS < 2**31 <= 384 * 32 * (XTB_MAX_KSTEPS + 4)
    assert xtb_plan(129, 65537, 132) == (31, 68, 2052)  # 2052 = 30 * 68 + 12: a short last split
    assert xtb_plan(300, 3000, 132)[0] == 1
    # the cap binds only past 174,760 k-steps (5.6 M variants) in one split, e.g. 25.6 M variants on more 128-sample
    # tiles than 2 SMs' worth
    assert xtb_plan(128 * 300, 32 * 800000, 132) == (5, XTB_MAX_KSTEPS, 800000)


# ------------------------------------------------------------------------------------------------------- device: XA
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 4, 127, 128, 129, 255, 256, 257])
def test_xa_sample_edges(gpu_ctx, n):
    """128 samples per staged k-block, the 64-sample digit blocks, 1..3 samples (fewer than 2k(k + 1))."""
    geno = _geno(300, n, seed=10 + n, mono_every=29)
    _products(gpu_ctx, geno, g=_dense(n, 3, n), h=_dense(300, 2, n + 1))


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 127, 128, 129])
def test_xa_variant_edges(gpu_ctx, m):
    """128 variants per XA CTA; the variant padding decodes as missing."""
    geno = _geno(m, 200, seed=20 + m)
    _products(gpu_ctx, geno, g=_dense(200, 4, m), h=_dense(m, 3, m + 1))


@pytest.mark.gpu
@pytest.mark.parametrize("cx", [1, 2, 31, 32, 33, 64, 65])
def test_column_group_edges(gpu_ctx, cx):
    """32 columns per launch: one, two and three column groups, full and partial, in both products."""
    geno = _geno(260, 140, seed=30 + cx, mono_every=41)
    _products(gpu_ctx, geno, g=_dense(140, cx, cx), h=_dense(260, cx, cx + 100))


@pytest.mark.gpu
def test_per_column_magnitudes(gpu_ctx):
    """Each column has its own scale: magnitudes 2^+-40 apart, an all-zero column (scale 1), one dominant entry."""
    n, m = 150, 400
    geno = _geno(m, n, seed=41)
    g = _dense(n, 6, 42) * np.array([1.0, 2.0**40, 2.0**-40, 0.0, 1.0, 2.0**-20])
    g[:, 3] = 0.0
    g[17, 4] = 2.0**35
    h = _dense(m, 6, 43) * np.array([2.0**-40, 1.0, 2.0**40, 0.0, 1.0, 3.0])
    h[:, 3] = 0.0
    h[201, 4] = -(2.0**35)
    _products(gpu_ctx, geno, g=g, h=h)


@pytest.mark.gpu
def test_degenerate_inputs(gpu_ctx):
    """Monomorphic variants (slope 0), an all-missing sample, an all-missing variant, given REF frequencies mixed with
    NaN (the variant's own count)."""
    n, m = 170, 500
    geno = _geno(m, n, seed=51, mono_every=23)
    geno[:, 9] = 3
    geno[77] = 3
    rng = np.random.default_rng(52)
    rf = rng.uniform(0.1, 0.9, size=m)
    rf[rng.random(m) < 0.4] = np.nan
    rf[0::23] = np.nan
    rf[11::23] = np.nan
    rf[77] = np.nan
    sl, _ = standardise(geno, rf)
    assert (sl == 0).sum() >= 40 and sl[77] > 0
    _products(gpu_ctx, geno, g=_dense(n, 5, 53), h=_dense(m, 5, 54), ref_freq=rf)


@pytest.mark.gpu
def test_chunked_uploads(gpu_ctx):
    """One add_variants call of 65,537 variants (two standardisation chunks), then odd-sized calls into one job."""
    geno = _geno(CHUNK + 1, 40, seed=61, mono_every=101)
    _products(gpu_ctx, geno, g=_dense(40, 3, 62), h=_dense(CHUNK + 1, 3, 63))
    calls = [1, 127, CHUNK + 3, 300]
    geno = _geno(sum(calls), 33, seed=64, mono_every=97)
    rf = np.where(np.random.default_rng(65).random(sum(calls)) < 0.5, np.nan, 0.3)
    rf[0::97] = np.nan
    rf[48::97] = np.nan
    _products(gpu_ctx, geno, g=_dense(33, 2, 66), h=_dense(sum(calls), 2, 67), ref_freq=rf, calls=calls)


# ------------------------------------------------------------------------------------------------------ device: XtB
@pytest.mark.gpu
@pytest.mark.parametrize("plan", ["one_split", "short_last_split", "tiles_over_2sm"])
def test_xtb_split_plans(gpu_ctx, plan):
    """The split-K plan depends on the SM count; each case picks (n, m) for the plan it names and asserts it."""
    sms = _sm_count()
    if plan == "one_split":
        n, m = 300, 3000  # 96 k-steps: fewer than two splits of 64
    elif plan == "short_last_split":
        n, m = 129, CHUNK + 1
    else:
        n, m = 128 * (2 * sms + 2) + 1, 4100  # more 128-sample tiles than 2 SMs' worth: one split from the SM term
    splits, kps, ksteps = xtb_plan(n, m, sms)
    if plan == "one_split":
        assert splits == 1 and ksteps // 64 == 1
    elif plan == "short_last_split":
        assert splits > 1 and ksteps % kps != 0 and -(-n // 128) < 2 * sms
    else:
        assert splits == 1 and ksteps // 64 > 1 and -(-n // 128) > 2 * sms
    geno = _geno(m, n, seed=70 + m, miss=0.02, mono_every=53)
    assert _products(gpu_ctx, geno, g=_dense(n, 2, 71), h=_dense(m, 2, 72), sms=sms) == splits


# ---------------------------------------------------------------------------------------- device: --pca approx
def _structured_geno(m, n, seed, pops, fst=0.2, miss=0.01):
    rng = np.random.default_rng(seed)
    anc = rng.uniform(0.1, 0.9, size=m)
    pf = rng.beta((anc * (1 - fst) / fst)[:, None], ((1 - anc) * (1 - fst) / fst)[:, None], size=(m, pops))
    f = pf[:, np.arange(n) % pops]
    g = (rng.random((m, n)) < f).astype(np.uint8) + (rng.random((m, n)) < f).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _align(vecs, ref):
    s = np.sign(np.sum(vecs * ref, axis=1, keepdims=True))
    s[s == 0] = 1
    return vecs * s


@pytest.mark.gpu
@pytest.mark.parametrize("n,m,k", [(12, 3000, 2), (13, 3000, 2), (129, 4000, 3), (257, 4000, 3), (300, CHUNK + 4464, 3)])
def test_pca_approx_edges(gpu_ctx, n, m, k):
    """The smallest allowed sample count n = 2k(k + 1) and one more, 129 / 257 samples, and more variants than one
    standardisation chunk; k + 1 populations so all k PCs are structure PCs."""
    geno = _structured_geno(m, n, seed=n + m, pops=k + 1)
    g1 = np.random.default_rng(n).standard_normal((n, 2 * k))
    want_vals, want_vecs = orc.pca_approx(geno, k, g1)
    vals, vecs = host.pca_approx(gpu_ctx, pack_genotypes(geno), n, k, g1)
    assert np.allclose(vals, want_vals, rtol=1e-6)
    assert np.allclose(_align(vecs, want_vecs), want_vecs, atol=1e-5 * np.abs(want_vecs).max())


# ---------------------------------------------------------------------------------------- device: --variant-score
def _vscores(ctx, geno, w, ref_freq=None):
    got = host.variant_scores(ctx, pack_genotypes(geno), geno.shape[1], w, ref_freqs=ref_freq)
    rf = filled_freqs(geno, ref_freq)
    _check(got, vscore_reference(geno, w, rf), vscore_bound(geno, w, rf), f"vscore n={geno.shape[1]} m={geno.shape[0]} cols={w.shape[1]}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 4, 129])
@pytest.mark.parametrize("cols", [1, 32, 33, 65])
def test_variant_score_shapes(gpu_ctx, n, cols):
    """Any sample count (VscoreReport has no minimum) and one to three weight-column groups."""
    geno = _geno(129, n, seed=80 + n, miss=0.1, mono_every=13)
    _vscores(gpu_ctx, geno, _dense(n, cols, cols))


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, CHUNK + 1])
def test_variant_score_variant_counts(gpu_ctx, m):
    geno = _geno(m, 37, seed=90, miss=0.1, mono_every=29)
    _vscores(gpu_ctx, geno, _dense(37, 3, 91))


@pytest.mark.gpu
def test_variant_score_frequencies_0_and_1(gpu_ctx):
    """Given ALT frequencies of exactly 0 and 1 on polymorphic variants with missing calls are used as given: the
    missing calls count 0 or 2, the called dosages count as they are (no zero-variance check, no slope)."""
    n, m = 60, 300
    geno = _geno(m, n, seed=95, miss=0.15, mono_every=31)
    rf = np.full(m, np.nan)
    rf[1::4] = 1.0  # ALT frequency 0
    rf[2::4] = 0.0  # ALT frequency 1
    assert (geno[1::4] == 1).any() and (geno[2::4] == 3).any()
    _vscores(gpu_ctx, geno, _dense(n, 3, 96), ref_freq=rf)


@pytest.mark.gpu
def test_variant_score_weight_span(gpu_ctx):
    """A weight column spanning 2^20 in magnitude next to an ordinary one: the bound is relative to the column maximum."""
    n, m = 129, 200
    geno = _geno(m, n, seed=97, miss=0.05)
    rng = np.random.default_rng(98)
    w = np.stack([rng.choice([-1.0, 1.0], n) * np.ldexp(1.0, rng.integers(0, 21, n)) * rng.uniform(1, 2, n), rng.standard_normal(n)], axis=1)
    assert np.abs(w[:, 0]).max() / np.abs(w[:, 0]).min() > 2.0**19
    _vscores(gpu_ctx, geno, w)


# ---------------------------------------------------------------------------------------------- device: CLI
def _table(path):
    rows = [ln.rstrip("\n").split("\t") for ln in open(path)]
    return rows[0], rows[1:]


def _cli_vs_golden(golden_dir, tmp_path, extra, golden):
    out = str(tmp_path / "v")
    r = subprocess.run([BIN, "--bfile", os.path.join(golden_dir, "v3"), *extra, "--variant-score", os.path.join(golden_dir, "v3_w.txt"), *(["cols=+altfreq"] if extra else []), "--out", out],
                       capture_output=True, text=True, env=ENV)
    assert r.returncode == 0, r.stdout + r.stderr
    got_h, got = _table(out + ".vscore")
    ref_h, ref = _table(os.path.join(golden_dir, golden))
    assert got_h == ref_h and len(got) == len(ref)
    first = ref_h.index("W1")
    for g, w in zip(got, ref):
        assert g[:first] == w[:first]
        for col in range(first, len(ref_h)):
            assert np.isclose(float(g[col]), float(w[col]), rtol=2e-5, atol=1e-12), (g, w)


@pytest.mark.gpu
def test_variant_score_cli_three_samples(golden_dir, tmp_path):
    """3 samples (fewer than any approx-PCA job allows), monomorphic and all-missing variants: the reference's report."""
    _cli_vs_golden(golden_dir, tmp_path, [], "v3.vscore")


@pytest.mark.gpu
def test_variant_score_cli_read_freq_0_and_1(golden_dir, tmp_path):
    """--read-freq gives ALT frequencies 0 and 1 to polymorphic variants with missing calls: the reference's report."""
    _cli_vs_golden(golden_dir, tmp_path, ["--read-freq", os.path.join(golden_dir, "v3_rf.afreq")], "v3_rf.vscore")


@pytest.mark.gpu
def test_variant_score_cli_crosses_a_job_boundary(tmp_path):
    """262,145 variants x 8 samples: two jobs of RunVscore, the second with one variant."""
    n, m = 8, VSCORE_PIECE + 1
    geno = _geno(m, n, seed=99, miss=0.1, mono_every=1001)
    code = np.array([3, 2, 0, 1], dtype=np.uint8)[geno]  # ALT dosage / missing -> .bed code
    q = np.concatenate([code, np.zeros((m, (-n) % 4), dtype=np.uint8)], axis=1).reshape(m, -1, 4)
    pre = str(tmp_path / "big")
    with open(pre + ".bed", "wb") as f:
        f.write(bytes([0x6C, 0x1B, 0x01]) + (q[..., 0] | (q[..., 1] << 2) | (q[..., 2] << 4) | (q[..., 3] << 6)).astype(np.uint8).tobytes())
    with open(pre + ".bim", "w") as f:
        f.write("".join(f"1\tb{k}\t0\t{k + 1}\tA\tG\n" for k in range(m)))
    with open(pre + ".fam", "w") as f:
        f.write("".join(f"f{k}\ti{k}\t0\t0\t0\t-9\n" for k in range(n)))
    w = np.round(_dense(n, 2, 100), 3)
    with open(pre + "_w.txt", "w") as f:
        f.write("#FID\tIID\tA\tB\n" + "".join(f"f{k}\ti{k}\t{float(w[k, 0])!r}\t{float(w[k, 1])!r}\n" for k in range(n)))
    r = subprocess.run([BIN, "--bfile", pre, "--variant-score", pre + "_w.txt", "--out", pre], capture_output=True, text=True, env=ENV)
    assert r.returncode == 0, r.stdout + r.stderr
    hdr, rows = _table(pre + ".vscore")
    assert hdr[-2:] == ["A", "B"] and len(rows) == m
    got = np.array([[float(x) for x in row[-2:]] for row in rows])
    want = orc.variant_scores(geno, w, orc.ref_allele_freqs(geno))
    assert np.allclose(got, want, rtol=2e-5, atol=1e-5 * np.abs(w).sum())
