"""GRM (grm_wg_kernel, grm.cu) at its tile, padding, staging and read-back edges against the fp64 oracle, under the
error bound of DESIGN §4 restated per entry.

The driver writes each batch's per-variant tables L1 = slope * z, L2 = intercept * z in fixed point with its own scale
2^F_b, F_b = 38 - e_b where 2^(e_b - 1) <= max |L| < 2^e_b over the batch's variants (grm.cu).  Rounding a table entry
costs at most 2^-(F_b + 1), and an entry of Z^T Z reads one L1 entry (times a dosage <= 2) and one L2 entry (times an
indicator <= 1) per variant, so a batch of n_b variants moves it by at most 3 n_b 2^-(F_b + 1).  Both sides then sum in
fp64; gamma_k (|Z|^T |Z|)_ij with k = M + batches + 3 covers the oracle's summation, the device's int64 -> fp64
conversions and cross-batch adds, and the final divisions.  Every entry of the lower triangle is held to
(sum_b 3 n_b 2^-(F_b + 1) + gamma_k (|Z|^T |Z|)_ij) / obs_ij, or that sum / M where the reference divides by the
variant count; observation counts are exact."""
import numpy as np
import pytest

from plink_ng_b200.host import GRM_COV, GRM_MEANIMPUTE, GrmJob, pack_genotypes, parallel_bounds
from oracle import plink_oracle as orc

FIXED_BITS = 38  # kGrmFixedBits: |L| 2^F < 2^38
STAGE_VARIANTS = 65536  # kMaxStageVariants: one add_variants call runs one launch per this many variants
UNIT = 2.0**-53


def _batches(calls):
    """[start, end) of every launch of a job whose add_variants calls pass `calls` variants each."""
    out, s = [], 0
    for ct in calls:
        for o in range(0, ct, STAGE_VARIANTS):
            k = min(STAGE_VARIANTS, ct - o)
            out.append((s, s + k))
            s += k
    return out


def _filled_freqs(geno, ref_freq):
    """The REF frequencies the driver uses: the given value, or the block's own count where it is NaN or absent."""
    own = orc.ref_allele_freqs(geno)
    return own if ref_freq is None else np.where(np.isnan(ref_freq), own, ref_freq)


def lookup_tables(geno, ref_freq=None, cov=False):
    """L1, L2 [M, 3] (genotype 0, 1, 2) as grm.cu builds them; zero rows for the variants it skips."""
    rf = _filled_freqs(geno, ref_freq)
    alt = 1.0 - rf
    if cov:
        skip = np.zeros(rf.shape, dtype=bool)
        inv = np.ones_like(rf)
    else:
        var = 2 * rf * alt
        skip = ~(var > orc.SMALL_EPSILON)
        inv = 1.0 / np.sqrt(np.where(skip, 1.0, var))
    slope, icpt = inv, -2 * alt * inv
    z = np.stack([icpt, icpt + slope, icpt + 2 * slope], axis=1)
    l1, l2 = slope[:, None] * z, icpt[:, None] * z
    l1[skip] = 0.0
    l2[skip] = 0.0
    return l1, l2


def batch_scales(l1, l2, calls):
    """F_b of every launch."""
    fs = []
    for s, e in _batches(calls):
        max_l = max(float(np.abs(l1[s:e]).max(initial=0.0)), float(np.abs(l2[s:e]).max(initial=0.0)))
        fs.append(FIXED_BITS - int(np.frexp(max_l)[1]) if max_l > 0.0 else 0)
    return fs


def _divisor(geno, meanimpute):
    """obs_ij (float, 0 where no variant is jointly observed) or M, as CalcGrm divides."""
    miss = geno == 3
    m = geno.shape[0]
    if meanimpute or not miss.any():
        return float(m)
    mf = miss.astype(np.float64)
    ct = miss.sum(axis=0).astype(np.float64)
    obs = m - ct[:, None] - ct[None, :] + np.rint(mf.T @ mf)
    np.fill_diagonal(obs, m - ct)
    return obs


def grm_error_bound(geno, calls, ref_freq=None, meanimpute=False, cov=False):
    """Per-entry bound on |G_device - G_oracle| [N, N] (inf where obs is 0) and the F_b of every launch."""
    l1, l2 = lookup_tables(geno, ref_freq, cov)
    calls = list(calls)
    fs = batch_scales(l1, l2, calls)
    fixed = sum(3.0 * (e - s) * 2.0 ** -(f + 1) for (s, e), f in zip(_batches(calls), fs))
    absz = np.abs(orc.centered_varmaj(geno, _filled_freqs(geno, ref_freq), not cov))
    k = geno.shape[0] + len(fs) + 3
    slack = fixed + (k * UNIT / (1 - k * UNIT)) * (absz.T @ absz)
    with np.errstate(divide="ignore"):
        return slack / _divisor(geno, meanimpute), fs


def emulate_fixed_point(geno, calls, ref_freq=None, meanimpute=False, cov=False, drop_d0=False):
    """The device's arithmetic in numpy: tables rounded to F_b bits per launch, exact integer contraction.
    drop_d0: the least significant base-256 digit of every table entry left out."""
    l1, l2 = lookup_tables(geno, ref_freq, cov)
    calls = list(calls)
    dos = np.where(geno == 3, 0, geno).astype(np.int64)
    nm = (geno != 3).astype(np.int64)
    n = geno.shape[1]
    acc = np.zeros((n, n))
    for (s, e), f in zip(_batches(calls), batch_scales(l1, l2, calls)):
        x1, x2 = (np.rint(t[s:e] * 2.0**f).astype(np.int64) for t in (l1, l2))
        if drop_d0:
            x1, x2 = (x - (((x + 128) & 255) - 128) for x in (x1, x2))
        part = np.zeros((n, n), dtype=np.int64)
        for c in range(3):
            sel = (geno[s:e] == c).astype(np.int64)
            part += dos[s:e].T @ (x1[:, c, None] * sel) + nm[s:e].T @ (x2[:, c, None] * sel)
        acc += part.astype(np.float64) * 2.0**-f
    with np.errstate(divide="ignore", invalid="ignore"):
        return acc / _divisor(geno, meanimpute)


def _geno(m, n, seed, miss=0.03, lo=0.02, mono_every=0):
    """Random hard calls; every `mono_every`-th variant monomorphic (alternately hom-REF and hom-ALT)."""
    rng = np.random.default_rng(seed)
    freq = rng.uniform(lo, 1 - lo, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    if mono_every:
        g[0::mono_every] = 0
        g[mono_every // 2 :: mono_every] = 2
    if miss:
        g[rng.random((m, n)) < miss] = 3
    return g


def _check(got, got_obs, want, obs, bound, r0, r1, block=512):
    """Lower triangle of rows [r0, r1): NaN exactly where the oracle has NaN, every other entry within its bound,
    observation counts exact."""
    for j0 in range(r0, r1, block):
        j1 = min(r1, j0 + block)
        jj, ii = np.tril_indices(j1)
        keep = jj >= j0
        jj, ii = jj[keep], ii[keep]
        a, b = got[jj - r0, ii], want[jj, ii]
        nan = np.isnan(b)
        assert np.array_equal(np.isnan(a), nan), (j0, j1)
        err, lim = np.abs(a[~nan] - b[~nan]), bound[jj, ii][~nan]
        bad = np.flatnonzero(~(err <= lim))
        assert bad.size == 0, f"{bad.size} entries of rows [{j0},{j1}) outside the bound, e.g. ({jj[~nan][bad[0]]},{ii[~nan][bad[0]]}): |err| {err[bad[0]]:.3g} > {lim[bad[0]]:.3g}"
        if obs is not None:
            assert np.array_equal(got_obs[jj - r0, ii], obs[jj, ii].astype(np.float32)), (j0, j1)


def _run(ctx, geno, calls=None, ref_freq=None, flags=0, r0=0, r1=None):
    """Job over rows [r0, r1), one add_variants call per entry of `calls`; returns rows, obs, oracle, bound, F_b."""
    m, n = geno.shape
    calls = [m] if calls is None else calls
    assert sum(calls) == m
    r1 = n if r1 is None else r1
    gv = pack_genotypes(geno)
    with GrmJob(ctx, n, r0, r1, flags) as job:
        s = 0
        for ct in calls:
            job.add_variants(gv[s : s + ct], ref_freqs=None if ref_freq is None else ref_freq[s : s + ct])
            s += ct
        got, got_obs = job.rows(with_obs=True)
    mi, cv = bool(flags & GRM_MEANIMPUTE), bool(flags & GRM_COV)
    want, obs = orc.grm(geno, ref_freq=None if ref_freq is None else _filled_freqs(geno, ref_freq), meanimpute=mi, cov=cv)
    bound, fs = grm_error_bound(geno, calls, ref_freq, meanimpute=mi, cov=cv)
    return got, got_obs, want, obs, bound, fs


# ------------------------------------------------------------------------------------------ the bound itself (CPU)
@pytest.mark.parametrize("flags", [0, GRM_COV])
def test_error_bound_holds_for_rounded_tables_and_catches_a_lost_digit(flags):
    """The numpy restatement of the device arithmetic stays inside the bound; the same arithmetic without the least
    significant digit D_0 does not, so the bound detects that defect."""
    geno = _geno(420, 48, seed=11, lo=0.2, mono_every=9)
    for v in range(151, 270, 7):  # singletons in the middle batch: its scale differs from its neighbours'
        geno[v] = np.where(geno[v] == 3, 3, 0)
        geno[v, v % 48] = 1
    calls = [150, 120, 150]
    mi, cv = False, bool(flags & GRM_COV)
    want, _ = orc.grm(geno, meanimpute=mi, cov=cv)
    bound, fs = grm_error_bound(geno, calls, meanimpute=mi, cov=cv)
    assert cv or len(set(fs)) > 1  # with GRM_COV every |L| is at most 4: one scale
    rows = np.tril_indices(48)
    err = np.abs(emulate_fixed_point(geno, calls, meanimpute=mi, cov=cv) - want)[rows]
    assert np.all(err <= bound[rows])
    assert err.max() > 0.0
    err_d0 = np.abs(emulate_fixed_point(geno, calls, meanimpute=mi, cov=cv, drop_d0=True) - want)[rows]
    assert np.any(err_d0 > bound[rows])


def test_batch_split_follows_the_staging_capacity():
    assert _batches([STAGE_VARIANTS + 257]) == [(0, STAGE_VARIANTS), (STAGE_VARIANTS, STAGE_VARIANTS + 257)]
    assert _batches([3, STAGE_VARIANTS]) == [(0, 3), (3, STAGE_VARIANTS + 3)]


# ------------------------------------------------------------------------------------------------------- device
@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 79, 80, 81, 127, 128, 129, 159, 160, 161, 639, 640, 641, 1281])
def test_grm_sample_count_edges(gpu_ctx, n):
    """Row tiles of 128, column tiles of 80, the 640-sample padding block and the sample-major copy past it;
    monomorphic variants stay in as zero columns that count in M and in obs."""
    geno = _geno(600, n, seed=100 + n, mono_every=25)
    got, got_obs, want, obs, bound, _ = _run(gpu_ctx, geno)
    assert obs is not None
    _check(got, got_obs, want, obs, bound, 0, n)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 63, 64, 65, 255, 256, 257, 513])
def test_grm_variant_count_edges(gpu_ctx, m):
    """64-variant stages and the 256-variant padding of a launch."""
    geno = _geno(m, 161, seed=200 + m, mono_every=31)
    geno[0, 0] = 3  # obs counts in use at every m
    got, got_obs, want, obs, bound, _ = _run(gpu_ctx, geno)
    _check(got, got_obs, want, obs, bound, 0, 161)


@pytest.mark.gpu
def test_grm_one_call_over_the_staging_capacity(gpu_ctx):
    """65,536 + 257 variants in one add_variants call: two launches, each with its own fixed-point scale."""
    geno = _geno(STAGE_VARIANTS + 257, 96, seed=31, lo=0.2, mono_every=97)
    tail = geno[STAGE_VARIANTS:]
    tail[::3] = np.where(tail[::3] == 3, 3, 0)  # rare variants in the second launch only: a coarser scale there
    tail[::3, 5] = 1
    got, got_obs, want, obs, bound, fs = _run(gpu_ctx, geno)
    assert len(fs) == 2 and fs[0] != fs[1]
    _check(got, got_obs, want, obs, bound, 0, 96)


@pytest.mark.gpu
def test_grm_batches_with_different_scales(gpu_ctx):
    """Common variants, then a batch with singletons, then common again: F_b differs between launches."""
    geno = _geno(700, 150, seed=41, lo=0.2)
    mid = geno[300:500]
    mid[::2] = np.where(mid[::2] == 3, 3, 0)
    mid[::2, 7] = 1
    got, got_obs, want, obs, bound, fs = _run(gpu_ctx, geno, calls=[300, 200, 200])
    assert fs[1] < fs[0] and fs[1] < fs[2]
    _check(got, got_obs, want, obs, bound, 0, 150)


@pytest.mark.gpu
@pytest.mark.parametrize("piece", [0, 1, 2, 3])
def test_grm_parallel_row_pieces(gpu_ctx, piece):
    """The four equal-area row pieces of 1,300 samples: they start inside 128-row tiles and cross the 640 block."""
    n = 1300
    r0, r1 = parallel_bounds(n, 0, piece, 4)
    geno = _geno(400, n, seed=51, mono_every=40)
    got, got_obs, want, obs, bound, _ = _run(gpu_ctx, geno, r0=r0, r1=r1)
    _check(got, got_obs, want, obs, bound, r0, r1)


@pytest.mark.gpu
def test_grm_row_subranges_of_one_job(gpu_ctx):
    n = 1300
    geno = _geno(300, n, seed=52, mono_every=40)
    want, obs = orc.grm(geno)
    bound, _ = grm_error_bound(geno, [300])
    with GrmJob(gpu_ctx, n) as job:
        job.add_variants(pack_genotypes(geno))
        for r0, r1 in ((0, 1), (5, 6), (127, 129), (130, 143), (600, 700), (639, 641), (1279, 1300), (0, n)):
            got, got_obs = job.rows(r0, r1, with_obs=True)
            _check(got, got_obs, want, obs, bound, r0, r1)


@pytest.mark.gpu
def test_grm_host_readback_split(gpu_ctx):
    """4,900 samples with obs: the 256 MiB read-back staging holds 2^28 / (12 * 4900) = 4,565 rows, so the copy
    splits inside a 128-row tile and inside a 16-row finalize block."""
    n = 4900
    assert (256 << 20) // (12 * n) == 4565
    geno = _geno(256, n, seed=61, mono_every=50)
    got, got_obs, want, obs, bound, _ = _run(gpu_ctx, geno)
    _check(got, got_obs, want, obs, bound, 0, n)


@pytest.mark.gpu
def test_grm_degenerate_inputs(gpu_ctx):
    """A sample missing everywhere (obs 0: NaN like the oracle's 0/0), two samples never observed together, an
    all-missing variant, and given REF frequencies mixed with NaN (the variant's own count)."""
    n, m = 200, 300
    geno = _geno(m, n, seed=71, mono_every=23)
    geno[:, 5] = 3
    geno[:150, 10] = 3
    geno[150:, 140] = 3
    geno[7] = 3
    rng = np.random.default_rng(72)
    rf = rng.uniform(0.1, 0.9, size=m)
    rf[rng.random(m) < 0.4] = np.nan
    rf[7] = np.nan
    rf[0::23] = np.nan  # monomorphic variants: their own (degenerate) frequency
    rf[11::23] = np.nan
    got, got_obs, want, obs, bound, _ = _run(gpu_ctx, geno, ref_freq=rf)
    assert obs[5, 5] == 0 and obs[140, 10] == 0 and np.isnan(want[140, 10])
    _check(got, got_obs, want, obs, bound, 0, n)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [GRM_COV, GRM_MEANIMPUTE, GRM_COV | GRM_MEANIMPUTE])
def test_grm_flags_past_the_padding_block(gpu_ctx, flags):
    n = 641
    geno = _geno(600, n, seed=81 + flags, mono_every=25)
    got, got_obs, want, obs, bound, _ = _run(gpu_ctx, geno, flags=flags)
    assert (obs is None) == bool(flags & GRM_MEANIMPUTE)
    _check(got, got_obs, want, obs, bound, 0, n)
