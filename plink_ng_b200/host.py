"""Thin host-side mirror of the reference's calling conventions for tests and bench.py.

Names follow the reference: `parallel_bounds` is ParallelBounds (2.0/plink2_common.cc:4956),
genotype blocks are "genovecs" in PgrGet layout (2.0/include/pgenlib_read.h:537), KING results are
`king_counts[pair][5]` (2.0/plink2_matrix_calc.cc:864-868).
"""
import ctypes as C
import math

import numpy as np

from . import capi
from .capi import lib, check

KING_ALGO_AUTO, KING_ALGO_POPCOUNT, KING_ALGO_TENSOR, KING_ALGO_TENSOR_TS = 0, 1, 2, 3


def pack_genotypes(geno: np.ndarray) -> np.ndarray:
    """[variants, samples] uint8 codes (0,1,2 = ALT dosage, 3 = missing) -> genovecs
    [variants, ceil(samples/32)] uint64 in PgrGet layout (trailing entries zero)."""
    geno = np.ascontiguousarray(geno, dtype=np.uint8)
    m, n = geno.shape
    n32 = (n + 31) // 32 * 32
    pad = np.zeros((m, n32), dtype=np.uint8)
    pad[:, :n] = geno & 3
    q = pad.reshape(m, n32 // 4, 4)
    by = (q[:, :, 0] | (q[:, :, 1] << 2) | (q[:, :, 2] << 4) | (q[:, :, 3] << 6)).astype(np.uint8)
    return np.ascontiguousarray(by).view("<u8").reshape(m, n32 // 32)


def unpack_genotypes(genovecs: np.ndarray, sample_ct: int) -> np.ndarray:
    by = np.ascontiguousarray(genovecs).view(np.uint8).reshape(genovecs.shape[0], -1)
    codes = np.stack([(by >> s) & 3 for s in (0, 2, 4, 6)], axis=-1).reshape(by.shape[0], -1)
    return np.ascontiguousarray(codes[:, :sample_ct])


def _triangle_divide(cur_prod_x2: int, modif: int) -> int:
    # 2.0/plink2_common.cc:4936-4954
    if cur_prod_x2 == 0:
        return -modif if modif < 0 else 0
    vv = int(math.sqrt(float(cur_prod_x2)))
    while (vv - 1) * (vv + modif - 1) >= cur_prod_x2:
        vv -= 1
    while vv * (vv + modif) < cur_prod_x2:
        vv += 1
    return vv


def parallel_bounds(ct: int, start: int, parallel_idx: int, parallel_tot: int):
    """ParallelBounds (2.0/plink2_common.cc:4956-4961): equal-area row range of piece k of n."""
    modif = 1 - start * 2
    ct_tot = ct * (ct + modif)
    return (
        _triangle_divide((ct_tot * parallel_idx) // parallel_tot, modif),
        _triangle_divide((ct_tot * (parallel_idx + 1)) // parallel_tot, modif),
    )


class GpuContext:
    def __init__(self, device_idx: int = 0):
        self._h = C.c_void_p()
        check(lib.pl2gpu_ctx_create(device_idx, C.byref(self._h)), "pl2gpu_ctx_create")

    @property
    def handle(self):
        return self._h

    def synchronize(self):
        check(lib.pl2gpu_ctx_synchronize(self._h), "pl2gpu_ctx_synchronize")

    def launch_count(self) -> int:
        return int(lib.pl2gpu_ctx_launch_count(self._h))

    def event_record(self, slot: int):
        check(lib.pl2gpu_ctx_event_record(self._h, slot), "pl2gpu_ctx_event_record")

    def event_elapsed_ms(self, slot_from: int, slot_to: int) -> float:
        ms = C.c_float()
        check(lib.pl2gpu_ctx_event_elapsed_ms(self._h, slot_from, slot_to, C.byref(ms)), "pl2gpu_ctx_event_elapsed_ms")
        return float(ms.value)

    def stream(self) -> int:
        return int(lib.pl2gpu_ctx_stream(self._h) or 0)

    def int8_peak(self, n_cols: int = 96, form: int = 1, min_seconds: float = 2.0):
        """Measured chip-wide wgmma rate (TOP/s, seconds): form 1 int8 (the roofline denominator), form 2 binary AND-POPC."""
        tops, secs = C.c_double(), C.c_double()
        check(lib.pl2gpu_int8_peak(self._h, n_cols, form, min_seconds, C.byref(tops), C.byref(secs)), "pl2gpu_int8_peak")
        return float(tops.value), float(secs.value)

    def bulk_read_rate(self, working_set_bytes: int, inflight_bytes: int, min_seconds: float = 0.5):
        """Measured bulk-copy read rate (TB/s, seconds) with inflight_bytes of copies in flight per SM."""
        tbps, secs = C.c_double(), C.c_double()
        check(lib.pl2gpu_bulk_read_rate(self._h, working_set_bytes, inflight_bytes, min_seconds, C.byref(tbps), C.byref(secs)), "pl2gpu_bulk_read_rate")
        return float(tbps.value), float(secs.value)

    def comm_init(self, rank: int, world: int, unique_id: bytes):
        """Attach an NCCL communicator (collective over all ranks; rank 0 makes the id with comm_unique_id())."""
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        check(lib.pl2gpu_comm_init(self._h, rank, world, buf), "pl2gpu_comm_init")

    def comm_destroy(self):
        """Collective teardown of the communicator (every rank calls it at the same point); idempotent."""
        check(lib.pl2gpu_comm_destroy(self._h), "pl2gpu_comm_destroy")

    def selftest_umma(self, verbose: bool = True):
        check(lib.pl2gpu_selftest_umma(self._h, 1 if verbose else 0), "pl2gpu_selftest_umma")

    def close(self):
        if self._h:
            lib.pl2gpu_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def comm_unique_id() -> bytes:
    buf = (C.c_uint8 * 128)()
    check(lib.pl2gpu_comm_unique_id(buf), "pl2gpu_comm_unique_id")
    return bytes(buf)


def _pairs(r0: int, r1: int, col_end: int = None) -> int:
    """Pairs (j, i) of rows [r0, r1) with i < j, and i < col_end when a column bound is given."""

    def tri(r):
        if col_end is None or r <= col_end:
            return r * (r - 1) // 2 if r else 0
        return col_end * (col_end - 1) // 2 + (r - col_end) * col_end

    return tri(r1) - tri(r0)


class KingJob:
    """CalcKing's dense loop (2.0/plink2_matrix_calc.cc:2016-2117) for one row range."""

    def __init__(self, ctx: GpuContext, sample_ct: int, row_start: int = 0, row_end: int = None, algo: int = KING_ALGO_AUTO, max_variants_per_add: int = 0):
        self.ctx = ctx
        self.sample_ct = sample_ct
        self.row_start = row_start
        self.row_end = sample_ct if row_end is None else row_end
        self.col_end = sample_ct
        self._h = C.c_void_p()
        check(lib.pl2gpu_king_begin_ex(ctx.handle, sample_ct, self.row_start, self.row_end, algo, max_variants_per_add, C.byref(self._h)), "pl2gpu_king_begin_ex")

    def add_variants(self, genovecs: np.ndarray):
        """genovecs: host uint64 [variants, ceil(sample_ct/32)] (PgrGet rows)."""
        g = np.ascontiguousarray(genovecs)
        assert g.dtype == np.uint64 and g.ndim == 2 and g.shape[1] * 32 >= self.sample_ct
        check(lib.pl2gpu_king_add_variants(self._h, g.ctypes.data, g.strides[0], g.shape[0], 0), "pl2gpu_king_add_variants")

    def add_variants_device(self, dev_ptr: int, stride_bytes: int, variant_ct: int, complete: bool = False):
        """complete=True: the device buffer is not being written by pending work (src_is_device = 2)."""
        check(lib.pl2gpu_king_add_variants(self._h, C.c_void_p(dev_ptr), stride_bytes, variant_ct, 2 if complete else 1), "pl2gpu_king_add_variants")

    def add_variants_sharded(self, ptr: int, stride_bytes: int, slice_variant_ct: int, src_is_device: int):
        """Collective: this rank's slice of the batch; the library all-gathers the column tile (NCCL)."""
        check(lib.pl2gpu_king_add_variants_sharded(self._h, C.c_void_p(ptr), stride_bytes, slice_variant_ct, src_is_device), "pl2gpu_king_add_variants_sharded")

    def last_kernel_ms(self) -> float:
        ms = C.c_float()
        check(lib.pl2gpu_king_last_kernel_ms(self._h, C.byref(ms)), "pl2gpu_king_last_kernel_ms")
        return float(ms.value)

    def last_planes(self, nbytes: int) -> np.ndarray:
        """The first nbytes of the column plane copy the last default-algorithm launch read (geno_tile.cuh)."""
        out = np.empty(nbytes, dtype=np.uint8)
        check(lib.pl2gpu_king_last_planes(self._h, out.ctypes.data, nbytes), "pl2gpu_king_last_planes")
        return out

    def counts(self, row_start: int = None, row_end: int = None) -> np.ndarray:
        r0 = self.row_start if row_start is None else row_start
        r1 = self.row_end if row_end is None else row_end
        out = np.empty((_pairs(r0, r1, self.col_end), 5), dtype=np.uint32)
        check(lib.pl2gpu_king_get_counts(self._h, r0, r1, out.ctypes.data, 0), "pl2gpu_king_get_counts")
        return out

    def kinship(self, row_start: int = None, row_end: int = None) -> np.ndarray:
        r0 = self.row_start if row_start is None else row_start
        r1 = self.row_end if row_end is None else row_end
        out = np.empty(_pairs(r0, r1, self.col_end), dtype=np.float64)
        check(lib.pl2gpu_king_get_kinship(self._h, r0, r1, out.ctypes.data, 0), "pl2gpu_king_get_kinship")
        return out

    def filtered(self, min_kinship: float, max_out: int = 1 << 20, row_start: int = None, row_end: int = None):
        """--king-table-filter on the device: (pairs [k,2] = (j, i), counts [k,5], kinship [k]) in table order,
        only pairs whose kinship is not below min_kinship.  Grows the buffers and retries on overflow."""
        r0 = self.row_start if row_start is None else row_start
        r1 = self.row_end if row_end is None else row_end
        while True:
            pairs = np.empty((max_out, 2), dtype=np.uint32)
            counts = np.empty((max_out, 5), dtype=np.uint32)
            kin = np.empty(max_out, dtype=np.float64)
            found = C.c_uint64(0)
            check(lib.pl2gpu_king_get_filtered(self._h, r0, r1, min_kinship, max_out, pairs.ctypes.data, counts.ctypes.data, kin.ctypes.data, C.byref(found)), "pl2gpu_king_get_filtered")
            if found.value <= max_out:
                k = found.value
                return pairs[:k], counts[:k], kin[:k]
            max_out = int(found.value)

    def counts_to_device(self, dev_ptr: int, row_start: int, row_end: int):
        check(lib.pl2gpu_king_get_counts(self._h, row_start, row_end, C.c_void_p(dev_ptr), 1), "pl2gpu_king_get_counts")

    def kinship_to_device(self, dev_ptr: int, row_start: int, row_end: int):
        check(lib.pl2gpu_king_get_kinship(self._h, row_start, row_end, C.c_void_p(dev_ptr), 1), "pl2gpu_king_get_kinship")

    def close(self):
        if self._h:
            lib.pl2gpu_king_end(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class MappedKingJob(KingJob):
    """pl2gpu_king_begin_mapped: KingJob over device positions, order[p] = sample index at position p (None = identity),
    rows [row_start, row_end), columns below col_end.  add_variants takes rows in sample-index order; every result is in
    positions ("1" = the smaller position)."""

    def __init__(self, ctx: GpuContext, sample_ct: int, order=None, row_start: int = 0, row_end: int = None, col_end: int = None, max_variants_per_add: int = 0):
        self.ctx = ctx
        self.sample_ct = sample_ct
        self.row_start = row_start
        self.row_end = sample_ct if row_end is None else row_end
        self.col_end = sample_ct if col_end is None else col_end
        self._h = C.c_void_p()
        self._order = None if order is None else np.ascontiguousarray(order, dtype=np.uint32)
        optr = None if self._order is None else self._order.ctypes.data
        check(lib.pl2gpu_king_begin_mapped(ctx.handle, sample_ct, optr, self.row_start, self.row_end, self.col_end, max_variants_per_add, C.byref(self._h)), "pl2gpu_king_begin_mapped")


class KingPairJob:
    """KING counts for an explicit pair list (`--king-table-subset`; CalcKingTableSubset,
    2.0/plink2_matrix_calc.cc:3224).  pairs: int array [P, 2] of sample indices (first, second)."""

    def __init__(self, ctx: GpuContext, sample_ct: int, pairs: np.ndarray):
        self.pairs = np.ascontiguousarray(pairs, dtype=np.uint32).reshape(-1, 2)
        self.sample_ct = sample_ct
        self._h = C.c_void_p()
        check(lib.pl2gpu_king_pairs_begin(ctx.handle, sample_ct, self.pairs.ctypes.data, len(self.pairs), C.byref(self._h)), "pl2gpu_king_pairs_begin")

    def add_variants(self, genovecs: np.ndarray):
        g = np.ascontiguousarray(genovecs)
        check(lib.pl2gpu_king_pairs_add_variants(self._h, g.ctypes.data, g.strides[0], g.shape[0], 0), "pl2gpu_king_pairs_add_variants")

    def counts(self) -> np.ndarray:
        out = np.empty((len(self.pairs), 5), dtype=np.uint32)
        check(lib.pl2gpu_king_pairs_get_counts(self._h, 0, len(self.pairs), out.ctypes.data, 0), "pl2gpu_king_pairs_get_counts")
        return out

    def close(self):
        if self._h:
            lib.pl2gpu_king_pairs_end(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def king_counts(genovecs: np.ndarray, sample_ct: int, algo: int = KING_ALGO_AUTO, device: int = 0, batch: int = 65536) -> np.ndarray:
    """All-pairs king_counts[pair][5] for one genotype block (convenience for tests)."""
    with GpuContext(device) as ctx, KingJob(ctx, sample_ct, 0, sample_ct, algo) as job:
        for s in range(0, genovecs.shape[0], batch):
            job.add_variants(genovecs[s : s + batch])
        return job.counts()


def geno_counts(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int) -> np.ndarray:
    """uint32 [variants, 4] = {hom-REF, het, hom-ALT, missing} (GenoarrCountFreqsUnsafe)."""
    g = np.ascontiguousarray(genovecs)
    out = np.empty((g.shape[0], 4), dtype=np.uint32)
    check(lib.pl2gpu_geno_counts(ctx.handle, g.ctypes.data, g.strides[0], sample_ct, g.shape[0], 0, out.ctypes.data), "pl2gpu_geno_counts")
    return out


def ld_band_flags(ctx: GpuContext, genovecs: np.ndarray, founder_ct: int, band: int, prune_ld_thresh: float) -> np.ndarray:
    g = np.ascontiguousarray(genovecs)
    out = np.zeros((g.shape[0], band), dtype=np.uint8)
    check(lib.pl2gpu_ld_band_flags(ctx.handle, g.ctypes.data, g.strides[0], founder_ct, g.shape[0], 0, band, prune_ld_thresh, out.ctypes.data), "pl2gpu_ld_band_flags")
    return out


def indep_pairwise(ctx: GpuContext, genovecs: np.ndarray, founder_ct: int, chr_codes, bps, window: int, step: int, r2: float, window_is_bp: bool = False, ref_freqs=None, preferred=None) -> np.ndarray:
    """LdPrune/IndepPairwise (2.0/plink2_ld.cc:2530) on an in-memory block -> removed[variants] uint8."""
    g = np.ascontiguousarray(genovecs)
    m = g.shape[0]
    chr_codes = np.ascontiguousarray(chr_codes, dtype=np.uint32)
    bps_a = np.ascontiguousarray(bps, dtype=np.uint32) if bps is not None else None
    rf = np.ascontiguousarray(ref_freqs, dtype=np.float64) if ref_freqs is not None else None
    pf = np.ascontiguousarray(preferred, dtype=np.uint8) if preferred is not None else None
    out = np.zeros(m, dtype=np.uint8)
    check(
        lib.pl2_indep_pairwise(ctx.handle, g.ctypes.data, g.strides[0], founder_ct, m, chr_codes.ctypes.data, bps_a.ctypes.data if bps_a is not None else None,
                               window, step, r2, 1 if window_is_bp else 0, rf.ctypes.data if rf is not None else None, pf.ctypes.data if pf is not None else None, 0, out.ctypes.data),
        "pl2_indep_pairwise",
    )
    return out


GRM_MEANIMPUTE, GRM_COV = 1, 2


class GrmJob:
    """CalcGrm's accumulation loop (2.0/plink2_matrix_calc.cc:4711-4749) for one row range."""

    def __init__(self, ctx: GpuContext, sample_ct: int, row_start: int = 0, row_end: int = None, flags: int = 0):
        self.ctx = ctx
        self.sample_ct = sample_ct
        self.row_start = row_start
        self.row_end = sample_ct if row_end is None else row_end
        self._h = C.c_void_p()
        check(lib.pl2gpu_grm_begin(ctx.handle, sample_ct, self.row_start, self.row_end, flags, C.byref(self._h)), "pl2gpu_grm_begin")

    def add_variants(self, genovecs: np.ndarray, ref_freqs=None):
        g = np.ascontiguousarray(genovecs)
        rf = None if ref_freqs is None else np.ascontiguousarray(ref_freqs, dtype=np.float64)
        rc = lib.pl2gpu_grm_add_variants(self._h, g.ctypes.data, g.strides[0], g.shape[0], 0, rf.ctypes.data if rf is not None else None)
        check(rc, "pl2gpu_grm_add_variants")

    def add_variants_device(self, dev_ptr: int, stride_bytes: int, variant_ct: int, ref_freqs=None):
        rf = None if ref_freqs is None else np.ascontiguousarray(ref_freqs, dtype=np.float64)
        check(lib.pl2gpu_grm_add_variants(self._h, C.c_void_p(dev_ptr), stride_bytes, variant_ct, 1, rf.ctypes.data if rf is not None else None), "pl2gpu_grm_add_variants")

    def rows(self, r0: int = None, r1: int = None, with_obs: bool = False):
        r0 = self.row_start if r0 is None else r0
        r1 = self.row_end if r1 is None else r1
        g = np.zeros((r1 - r0, r1), dtype=np.float64)
        obs = np.zeros((r1 - r0, r1), dtype=np.float32) if with_obs else None
        check(lib.pl2gpu_grm_get_rows(self._h, r0, r1, g.ctypes.data, obs.ctypes.data if with_obs else None, r1, 0), "pl2gpu_grm_get_rows")
        return (g, obs) if with_obs else g

    def eigen_topk(self, pc_ct: int):
        """Exact --pca: (eigvals[pc_ct] descending, eigvecs[pc_ct, samples])."""
        vals = np.empty(pc_ct, dtype=np.float64)
        vecs = np.empty((pc_ct, self.sample_ct), dtype=np.float64)
        check(lib.pl2gpu_grm_eigen_topk(self._h, pc_ct, vals.ctypes.data, vecs.ctypes.data), "pl2gpu_grm_eigen_topk")
        return vals, vecs

    def close(self):
        if self._h:
            lib.pl2gpu_grm_end(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def pca_approx(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, pc_ct: int, g1: np.ndarray, ref_freqs=None):
    """`--pca approx` on an in-memory block with a caller-supplied Gaussian start matrix
    g1 [sample_ct, 2*pc_ct] -> (eigvals[pc_ct], eigvecs[pc_ct, sample_ct])."""
    g = np.ascontiguousarray(genovecs)
    g1 = np.ascontiguousarray(g1, dtype=np.float64)
    assert g1.shape == (sample_ct, 2 * pc_ct)
    rf = None if ref_freqs is None else np.ascontiguousarray(ref_freqs, dtype=np.float64)
    h = C.c_void_p()
    check(lib.pl2gpu_pca_begin(ctx.handle, sample_ct, g.shape[0], pc_ct, C.byref(h)), "pl2gpu_pca_begin")
    try:
        check(lib.pl2gpu_pca_add_variants(h, g.ctypes.data, g.strides[0], g.shape[0], 0, rf.ctypes.data if rf is not None else None), "pl2gpu_pca_add_variants")
        vals = np.empty(pc_ct, dtype=np.float64)
        vecs = np.empty((pc_ct, sample_ct), dtype=np.float64)
        check(lib.pl2gpu_pca_run(h, g1.ctypes.data, vals.ctypes.data, vecs.ctypes.data), "pl2gpu_pca_run")
        return vals, vecs
    finally:
        lib.pl2gpu_pca_end(h)


def pca_products(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, g=None, h=None, ref_freqs=None, calls=None):
    """The two products of `--pca approx` (pl2gpu_pca_products) on the standardised matrix Y [variants, samples] of an
    in-memory block: g [sample_ct, cx] -> Y g [variants, cx]; h [variants, ct] -> Y^T h [sample_ct, ct].  calls: the
    variant counts of successive add_variants calls (default: one call).  Returns (Y g or None, Y^T h or None)."""
    gv = np.ascontiguousarray(genovecs)
    m = gv.shape[0]
    calls = [m] if calls is None else list(calls)
    assert sum(calls) == m
    rf = None if ref_freqs is None else np.ascontiguousarray(ref_freqs, dtype=np.float64)
    ga = None if g is None else np.ascontiguousarray(g, dtype=np.float64)
    ha = None if h is None else np.asfortranarray(h, dtype=np.float64)  # column-major [ct][variant]
    assert ga is None or ga.shape[0] == sample_ct
    assert ha is None or ha.shape[0] == m
    yg = None if ga is None else np.empty((ga.shape[1], m), dtype=np.float64)
    yth = None if ha is None else np.empty((sample_ct, ha.shape[1]), dtype=np.float64)
    job = C.c_void_p()
    check(lib.pl2gpu_pca_begin_shard(ctx.handle, sample_ct, m, 1, C.byref(job)), "pl2gpu_pca_begin_shard")
    try:
        s = 0
        for ct in calls:
            part = None if rf is None else rf[s : s + ct]
            check(lib.pl2gpu_pca_add_variants(job, gv[s:].ctypes.data, gv.strides[0], ct, 0, part.ctypes.data if part is not None else None), "pl2gpu_pca_add_variants")
            s += ct
        check(lib.pl2gpu_pca_products(job, ga.ctypes.data if ga is not None else None, 0 if ga is None else ga.shape[1], yg.ctypes.data if yg is not None else None,
                                      ha.ctypes.data if ha is not None else None, 0 if ha is None else ha.shape[1], yth.ctypes.data if yth is not None else None), "pl2gpu_pca_products")
        return (None if yg is None else yg.T), yth
    finally:
        lib.pl2gpu_pca_end(job)


def score_sums(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, weights4: np.ndarray, named_dosages: np.ndarray):
    """`--score` accumulation (pl2gpu_score_*) over an in-memory block of scored entries: genovecs [entries, words]
    PgrGet rows, weights4 [entries, 4] fp64 contributions of genotype codes 0..3, named_dosages [entries] uint8
    (dosages of codes 0, 1, 2 packed two bits each) -> (score sums, named-allele dosage sums, missing counts)."""
    g = np.ascontiguousarray(genovecs)
    w = np.ascontiguousarray(weights4, dtype=np.float64)
    d = np.ascontiguousarray(named_dosages, dtype=np.uint8)
    assert w.shape == (g.shape[0], 4) and d.shape == (g.shape[0],)
    h = C.c_void_p()
    check(lib.pl2gpu_score_begin(ctx.handle, sample_ct, C.byref(h)), "pl2gpu_score_begin")
    try:
        check(lib.pl2gpu_score_add_variants(h, g.ctypes.data, g.strides[0], g.shape[0], 0, w.ctypes.data, d.ctypes.data), "pl2gpu_score_add_variants")
        sums = np.empty(sample_ct, dtype=np.float64)
        dos = np.empty(sample_ct, dtype=np.uint64)
        miss = np.empty(sample_ct, dtype=np.uint32)
        check(lib.pl2gpu_score_get(h, sums.ctypes.data, dos.ctypes.data, miss.ctypes.data), "pl2gpu_score_get")
        return sums, dos, miss
    finally:
        lib.pl2gpu_score_end(h)


def score_sums_cols(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, weights4: np.ndarray, named_dosages: np.ndarray):
    """Several `--score` coefficient columns in one pass (pl2gpu_score_begin_cols): weights4 [entries, score_ct, 4] ->
    (score sums [sample_ct, score_ct], named-allele dosage sums, missing counts); otherwise as score_sums."""
    g = np.ascontiguousarray(genovecs)
    w = np.ascontiguousarray(weights4, dtype=np.float64)
    d = np.ascontiguousarray(named_dosages, dtype=np.uint8)
    assert w.ndim == 3 and w.shape[0] == g.shape[0] and w.shape[2] == 4 and d.shape == (g.shape[0],)
    score_ct = w.shape[1]
    h = C.c_void_p()
    check(lib.pl2gpu_score_begin_cols(ctx.handle, sample_ct, score_ct, C.byref(h)), "pl2gpu_score_begin_cols")
    try:
        check(lib.pl2gpu_score_add_variants(h, g.ctypes.data, g.strides[0], g.shape[0], 0, w.ctypes.data, d.ctypes.data), "pl2gpu_score_add_variants")
        sums = np.empty((sample_ct, score_ct), dtype=np.float64)
        dos = np.empty(sample_ct, dtype=np.uint64)
        miss = np.empty(sample_ct, dtype=np.uint32)
        check(lib.pl2gpu_score_get(h, sums.ctypes.data, dos.ctypes.data, miss.ctypes.data), "pl2gpu_score_get")
        return sums, dos, miss
    finally:
        lib.pl2gpu_score_end(h)


SCORE_DIPLOID, SCORE_HAPLOID_ALL, SCORE_CHR_Y, SCORE_CHR_X_MALE_HAPLOID = 0, 1, 2, 3  # kPl2Score* ploidy classes


def score_sums_ploidy(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, sample_sex: np.ndarray, ploidy_classes: np.ndarray, weights4_diploid: np.ndarray, weights4_haploid: np.ndarray, named_dosages: np.ndarray):
    """`--score` with sex-dependent ploidy (pl2gpu_score_set_sex / _add_variants_ploidy / _get_ploidy): sample_sex
    [sample_ct] (0 unknown, 1 male, 2 female), ploidy_classes [entries] (SCORE_*), both tables [entries, score_ct, 4]
    -> (score sums [sample_ct, score_ct], named-allele dosage sums in half allele units, diploid missing counts,
    haploid missing counts)."""
    g = np.ascontiguousarray(genovecs)
    wd = np.ascontiguousarray(weights4_diploid, dtype=np.float64)
    wh = np.ascontiguousarray(weights4_haploid, dtype=np.float64)
    pc = np.ascontiguousarray(ploidy_classes, dtype=np.uint8)
    sx = np.ascontiguousarray(sample_sex, dtype=np.uint8)
    d = np.ascontiguousarray(named_dosages, dtype=np.uint8)
    assert wd.ndim == 3 and wd.shape == wh.shape and wd.shape[0] == g.shape[0] and wd.shape[2] == 4 and d.shape == pc.shape == (g.shape[0],) and sx.shape == (sample_ct,)
    score_ct = wd.shape[1]
    h = C.c_void_p()
    check(lib.pl2gpu_score_begin_cols(ctx.handle, sample_ct, score_ct, C.byref(h)), "pl2gpu_score_begin_cols")
    try:
        check(lib.pl2gpu_score_set_sex(h, sx.ctypes.data), "pl2gpu_score_set_sex")
        check(lib.pl2gpu_score_add_variants_ploidy(h, g.ctypes.data, g.strides[0], g.shape[0], 0, pc.ctypes.data, wd.ctypes.data, wh.ctypes.data, d.ctypes.data), "pl2gpu_score_add_variants_ploidy")
        sums = np.empty((sample_ct, score_ct), dtype=np.float64)
        hdos = np.empty(sample_ct, dtype=np.uint64)
        miss_d = np.empty(sample_ct, dtype=np.uint32)
        miss_h = np.empty(sample_ct, dtype=np.uint32)
        check(lib.pl2gpu_score_get_ploidy(h, sums.ctypes.data, hdos.ctypes.data, miss_d.ctypes.data, miss_h.ctypes.data), "pl2gpu_score_get_ploidy")
        return sums, hdos, miss_d, miss_h
    finally:
        lib.pl2gpu_score_end(h)


def score_sums_classes(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, class_ct: int, entry_classes: np.ndarray, weights4_diploid: np.ndarray, named_dosages: np.ndarray, sample_sex=None, ploidy_classes=None,
                       weights4_haploid=None, batches=None):
    """`--score` into class_ct accumulator sets (pl2gpu_score_begin_classes / _add_variants_classes / _get_class):
    entry_classes [entries] (< class_ct), tables as score_sums_ploidy; ploidy_classes None scores every entry as
    diploid.  batches: entry counts of successive add calls (default: one call).  -> per class (score sums
    [sample_ct, score_ct], named-allele dosage sums in half allele units, diploid and haploid missing counts)."""
    g = np.ascontiguousarray(genovecs)
    wd = np.ascontiguousarray(weights4_diploid, dtype=np.float64)
    ec = np.ascontiguousarray(entry_classes, dtype=np.uint32)
    d = np.ascontiguousarray(named_dosages, dtype=np.uint8)
    assert wd.ndim == 3 and wd.shape[0] == g.shape[0] and wd.shape[2] == 4 and d.shape == ec.shape == (g.shape[0],)
    pc = None if ploidy_classes is None else np.ascontiguousarray(ploidy_classes, dtype=np.uint8)
    wh = None if weights4_haploid is None else np.ascontiguousarray(weights4_haploid, dtype=np.float64)
    score_ct = wd.shape[1]
    h = C.c_void_p()
    check(lib.pl2gpu_score_begin_classes(ctx.handle, sample_ct, score_ct, class_ct, C.byref(h)), "pl2gpu_score_begin_classes")
    try:
        if sample_sex is not None:
            sx = np.ascontiguousarray(sample_sex, dtype=np.uint8)
            check(lib.pl2gpu_score_set_sex(h, sx.ctypes.data), "pl2gpu_score_set_sex")
        e0 = 0
        for cnt in (batches or [g.shape[0]]):
            check(lib.pl2gpu_score_add_variants_classes(h, g[e0:].ctypes.data, g.strides[0], cnt, 0, ec[e0:].ctypes.data, None if pc is None else pc[e0:].ctypes.data, wd[e0:].ctypes.data,
                                                        None if wh is None else wh[e0:].ctypes.data, d[e0:].ctypes.data), "pl2gpu_score_add_variants_classes")
            e0 += cnt
        out = []
        for k in range(class_ct):
            sums = np.empty((sample_ct, score_ct), dtype=np.float64)
            hdos = np.empty(sample_ct, dtype=np.uint64)
            miss_d = np.empty(sample_ct, dtype=np.uint32)
            miss_h = np.empty(sample_ct, dtype=np.uint32)
            check(lib.pl2gpu_score_get_class(h, k, sums.ctypes.data, hdos.ctypes.data, miss_d.ctypes.data, miss_h.ctypes.data), "pl2gpu_score_get_class")
            out.append((sums, hdos, miss_d, miss_h))
        return out
    finally:
        lib.pl2gpu_score_end(h)


def score_sums_entries(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, class_ct: int, entry_rows: np.ndarray, entry_classes: np.ndarray, weights4_diploid: np.ndarray, named_dosages: np.ndarray, sample_sex=None,
                       ploidy_classes=None, weights4_haploid=None, batches=None):
    """`--score` entries that share staged rows (pl2gpu_score_begin_classes / _add_entries / _get_class): genovecs
    [rows, bytes]; entry_rows [entries] (non-decreasing row of each entry), entry_classes and the tables as
    score_sums_classes, per entry.  batches: row counts of successive add calls, each with the entries of its rows
    (default: one call).  -> per class (score sums [sample_ct, score_ct], named-allele dosage sums in half allele units,
    diploid and haploid missing counts)."""
    g = np.ascontiguousarray(genovecs)
    wd = np.ascontiguousarray(weights4_diploid, dtype=np.float64)
    er = np.ascontiguousarray(entry_rows, dtype=np.uint32)
    ec = np.ascontiguousarray(entry_classes, dtype=np.uint32)
    d = np.ascontiguousarray(named_dosages, dtype=np.uint8)
    assert wd.ndim == 3 and wd.shape[0] == er.shape[0] and wd.shape[2] == 4 and d.shape == ec.shape == er.shape
    pc = None if ploidy_classes is None else np.ascontiguousarray(ploidy_classes, dtype=np.uint8)
    wh = None if weights4_haploid is None else np.ascontiguousarray(weights4_haploid, dtype=np.float64)
    score_ct = wd.shape[1]
    h = C.c_void_p()
    check(lib.pl2gpu_score_begin_classes(ctx.handle, sample_ct, score_ct, class_ct, C.byref(h)), "pl2gpu_score_begin_classes")
    try:
        if sample_sex is not None:
            sx = np.ascontiguousarray(sample_sex, dtype=np.uint8)
            check(lib.pl2gpu_score_set_sex(h, sx.ctypes.data), "pl2gpu_score_set_sex")
        r0 = 0
        for cnt in (batches or [g.shape[0]]):
            e0, e1 = np.searchsorted(er, r0), np.searchsorted(er, r0 + cnt)
            rows = np.ascontiguousarray(er[e0:e1] - r0)
            check(lib.pl2gpu_score_add_entries(h, g[r0:].ctypes.data, g.strides[0], cnt, 0, int(e1 - e0), rows.ctypes.data, ec[e0:].ctypes.data, None if pc is None else pc[e0:].ctypes.data, wd[e0:].ctypes.data,
                                               None if wh is None else wh[e0:].ctypes.data, d[e0:].ctypes.data), "pl2gpu_score_add_entries")
            r0 += cnt
        out = []
        for k in range(class_ct):
            sums = np.empty((sample_ct, score_ct), dtype=np.float64)
            hdos = np.empty(sample_ct, dtype=np.uint64)
            miss_d = np.empty(sample_ct, dtype=np.uint32)
            miss_h = np.empty(sample_ct, dtype=np.uint32)
            check(lib.pl2gpu_score_get_class(h, k, sums.ctypes.data, hdos.ctypes.data, miss_d.ctypes.data, miss_h.ctypes.data), "pl2gpu_score_get_class")
            out.append((sums, hdos, miss_d, miss_h))
        return out
    finally:
        lib.pl2gpu_score_end(h)


def variant_scores(ctx: GpuContext, genovecs: np.ndarray, sample_ct: int, weights: np.ndarray, ref_freqs=None) -> np.ndarray:
    """`--variant-score` sums (pl2gpu_pca_vscore) for an in-memory block: weights [sample_ct, cols] -> [variants, cols]."""
    g = np.ascontiguousarray(genovecs)
    w = np.ascontiguousarray(weights, dtype=np.float64)
    assert w.shape[0] == sample_ct
    rf = None if ref_freqs is None else np.ascontiguousarray(ref_freqs, dtype=np.float64)
    h = C.c_void_p()
    check(lib.pl2gpu_pca_begin_shard(ctx.handle, sample_ct, g.shape[0], 0, C.byref(h)), "pl2gpu_pca_begin_shard")  # pc_ct 0: a --variant-score job
    try:
        check(lib.pl2gpu_pca_add_variants(h, g.ctypes.data, g.strides[0], g.shape[0], 0, rf.ctypes.data if rf is not None else None), "pl2gpu_pca_add_variants")
        out = np.empty((g.shape[0], w.shape[1]), dtype=np.float64)
        check(lib.pl2gpu_pca_vscore(h, w.ctypes.data, w.shape[1], out.ctypes.data), "pl2gpu_pca_vscore")
        return out
    finally:
        lib.pl2gpu_pca_end(h)
