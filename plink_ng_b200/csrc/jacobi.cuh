// jacobi.cuh - one-sided Jacobi (Hestenes) SVD of a column-major rows x q fp64 matrix, rows >= q.
//
// Used for the three dense factorizations of the PCA path (2.0/plink2_matrix_calc.cc): the top
// eigenpairs of the GRM (:5943-6039, dsyevr in the reference), the orthonormal basis of the Krylov
// matrix (:5860, dgesvd) and the final skinny SVD (:5920, dgesvd).  No library: the image's
// cuSOLVER + cuBLAS closure is ~2 GB of shared objects that take minutes to page in on a cold box.
//
// Columns are rotated pairwise until mutually orthogonal: A V = U Sigma.  Round-robin ordering gives
// q/2 disjoint pairs per round; a round is one launch (rows <= 8192: fused, both columns live in
// registers) or two (partial dot products per row chunk, then a deterministic fixed-order reduction
// + rotation), so results are bit-reproducible run to run.  Relative accuracy is that of Jacobi
// (small singular values included), which matters for the badly conditioned Krylov matrix.
// Cost per sweep ~ 3 q^2 rows fp64 flops, memory-bound; 6-12 sweeps.
#pragma once
#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

#include "common.cuh"

namespace pl2 {

constexpr uint32_t kJacobiThreads = 256;
constexpr uint32_t kJacobiFusedRows = 8192;  // 32 elements per thread per column
constexpr uint32_t kJacobiMaxChunks = 64;

struct JacobiRot {
  double c, s;
  bool rotate;
};

// Rotation that orthogonalises columns a, b given aa = a.a, bb = b.b, ab = a.b:  a' = c a - s b, b' = s a + c b.
__device__ __forceinline__ JacobiRot jacobi_rotation(double aa, double bb, double ab, double tol) {
  JacobiRot r;
  r.c = 1.0;
  r.s = 0.0;
  r.rotate = false;
  if (!(aa > 0.0) || !(bb > 0.0)) return r;
  if (fabs(ab) <= tol * sqrt(aa) * sqrt(bb)) return r;
  const double zeta = (bb - aa) / (2.0 * ab);
  const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
  r.c = 1.0 / sqrt(1.0 + t * t);
  r.s = r.c * t;
  r.rotate = true;
  return r;
}

__device__ __forceinline__ double block_sum(double v, double* red /* [kJacobiThreads / 32] */) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  const uint32_t w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  double tot = 0.0;
#pragma unroll
  for (uint32_t i = 0; i < kJacobiThreads / 32; ++i) tot += red[i];  // same order in every thread
  return tot;
}

// rows <= kJacobiFusedRows: one CTA per pair, columns held in registers.
static __global__ void __launch_bounds__(kJacobiThreads) jacobi_fused_kernel(double* __restrict__ a, uint64_t lda, uint32_t rows, const int2* __restrict__ pairs, double tol, int* __restrict__ rotated) {
  __shared__ double red[kJacobiThreads / 32];
  const int2 pr = pairs[blockIdx.x];
  if (pr.x < 0 || pr.y < 0) return;
  double* ca = a + static_cast<uint64_t>(pr.x) * lda;
  double* cb = a + static_cast<uint64_t>(pr.y) * lda;
  constexpr uint32_t kPer = kJacobiFusedRows / kJacobiThreads;
  double va[kPer], vb[kPer];
  double aa = 0.0, bb = 0.0, ab = 0.0;
#pragma unroll
  for (uint32_t e = 0; e < kPer; ++e) {
    const uint32_t r = e * kJacobiThreads + threadIdx.x;
    va[e] = (r < rows) ? ca[r] : 0.0;
    vb[e] = (r < rows) ? cb[r] : 0.0;
    aa = fma(va[e], va[e], aa);
    bb = fma(vb[e], vb[e], bb);
    ab = fma(va[e], vb[e], ab);
  }
  aa = block_sum(aa, red);
  bb = block_sum(bb, red);
  ab = block_sum(ab, red);
  const JacobiRot rot = jacobi_rotation(aa, bb, ab, tol);
  if (!rot.rotate) return;
  if (threadIdx.x == 0) *rotated = 1;
#pragma unroll
  for (uint32_t e = 0; e < kPer; ++e) {
    const uint32_t r = e * kJacobiThreads + threadIdx.x;
    if (r < rows) {
      ca[r] = rot.c * va[e] - rot.s * vb[e];
      cb[r] = rot.s * va[e] + rot.c * vb[e];
    }
  }
}

// tall matrices: partial dot products per (pair, row chunk) ...
static __global__ void __launch_bounds__(kJacobiThreads) jacobi_dots_kernel(const double* __restrict__ a, uint64_t lda, uint32_t rows, const int2* __restrict__ pairs, uint32_t chunk_rows, double* __restrict__ partial) {
  __shared__ double red[kJacobiThreads / 32];
  const int2 pr = pairs[blockIdx.x];
  if (pr.x < 0 || pr.y < 0) return;
  const double* ca = a + static_cast<uint64_t>(pr.x) * lda;
  const double* cb = a + static_cast<uint64_t>(pr.y) * lda;
  const uint32_t r0 = blockIdx.y * chunk_rows, r1 = min(rows, r0 + chunk_rows);
  double aa = 0.0, bb = 0.0, ab = 0.0;
  for (uint32_t r = r0 + threadIdx.x; r < r1; r += kJacobiThreads) {
    const double x = ca[r], y = cb[r];
    aa = fma(x, x, aa);
    bb = fma(y, y, bb);
    ab = fma(x, y, ab);
  }
  aa = block_sum(aa, red);
  bb = block_sum(bb, red);
  ab = block_sum(ab, red);
  if (threadIdx.x == 0) {
    double* p = partial + (static_cast<uint64_t>(blockIdx.x) * gridDim.y + blockIdx.y) * 3;
    p[0] = aa;
    p[1] = bb;
    p[2] = ab;
  }
}

// ... then every CTA of the pair reduces the partials in the same fixed order and rotates its chunk.
static __global__ void __launch_bounds__(kJacobiThreads) jacobi_rotate_kernel(double* __restrict__ a, uint64_t lda, uint32_t rows, const int2* __restrict__ pairs, uint32_t chunk_rows, const double* __restrict__ partial, double tol, int* __restrict__ rotated) {
  const int2 pr = pairs[blockIdx.x];
  if (pr.x < 0 || pr.y < 0) return;
  double aa = 0.0, bb = 0.0, ab = 0.0;
  const double* p = partial + static_cast<uint64_t>(blockIdx.x) * gridDim.y * 3;
  for (uint32_t ch = 0; ch < gridDim.y; ++ch) {
    aa += p[3 * ch];
    bb += p[3 * ch + 1];
    ab += p[3 * ch + 2];
  }
  const JacobiRot rot = jacobi_rotation(aa, bb, ab, tol);
  if (!rot.rotate) return;
  if (threadIdx.x == 0 && blockIdx.y == 0) *rotated = 1;
  double* ca = a + static_cast<uint64_t>(pr.x) * lda;
  double* cb = a + static_cast<uint64_t>(pr.y) * lda;
  const uint32_t r0 = blockIdx.y * chunk_rows, r1 = min(rows, r0 + chunk_rows);
  for (uint32_t r = r0 + threadIdx.x; r < r1; r += kJacobiThreads) {
    const double x = ca[r], y = cb[r];
    ca[r] = rot.c * x - rot.s * y;
    cb[r] = rot.s * x + rot.c * y;
  }
}

static __global__ void __launch_bounds__(kJacobiThreads) jacobi_colnorm_kernel(const double* __restrict__ a, uint64_t lda, uint32_t rows, double* __restrict__ norms) {
  __shared__ double red[kJacobiThreads / 32];
  const double* ca = a + static_cast<uint64_t>(blockIdx.x) * lda;
  double aa = 0.0;
  for (uint32_t r = threadIdx.x; r < rows; r += kJacobiThreads) aa = fma(ca[r], ca[r], aa);
  aa = block_sum(aa, red);
  if (threadIdx.x == 0) norms[blockIdx.x] = sqrt(aa);
}

// out[:, r] = a[:, perm[r]] / norm[perm[r]]   (zero column when the norm is zero)
static __global__ void jacobi_gather_kernel(const double* __restrict__ a, uint64_t lda, uint32_t rows, const uint32_t* __restrict__ perm, const double* __restrict__ norms, double* __restrict__ out, uint64_t ldo) {
  const uint32_t src = perm[blockIdx.y];
  const double nrm = norms[src];
  const double inv = nrm > 0.0 ? 1.0 / nrm : 0.0;
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) out[static_cast<uint64_t>(blockIdx.y) * ldo + r] = a[static_cast<uint64_t>(src) * lda + r] * inv;
}

// JacobiSvd after its shape check: the scratch is freed on return, before JacobiSvd clears the CUDA error state
static int JacobiSvdRun(Ctx* c, double* d_a, uint64_t lda, uint32_t rows, uint32_t q, uint32_t out_cols, double* sigma_host, double* d_u, uint64_t ldu, uint32_t* sweeps_out, const char** err) {
  const uint32_t qe = (q + 1) & ~1u;
  const uint32_t half = qe / 2, rounds = qe - 1;
  std::vector<int2> sched(static_cast<size_t>(rounds ? rounds : 1) * half);
  {
    std::vector<int> arr(qe);
    std::iota(arr.begin(), arr.end(), 0);
    for (uint32_t r = 0; r < rounds; ++r) {
      for (uint32_t i = 0; i < half; ++i) {
        int x = arr[i], y = arr[qe - 1 - i];
        if (x > y) std::swap(x, y);
        if (y >= static_cast<int>(q)) x = y = -1;  // phantom column of an odd q
        sched[static_cast<size_t>(r) * half + i] = make_int2(x, y);
      }
      std::rotate(arr.begin() + 1, arr.end() - 1, arr.end());  // player 0 fixed, the rest rotate
    }
  }
  const bool fused = rows <= kJacobiFusedRows;
  uint32_t chunk_rows = rows, chunks = 1;
  if (!fused) {
    chunk_rows = std::max<uint32_t>(16384, DivUpU32(rows, kJacobiMaxChunks));
    chunks = DivUpU32(rows, chunk_rows);
  }
  DevArray<int2> d_sched;
  DevArray<double> d_partial, d_norms;
  DevArray<uint32_t> d_perm;
  DevArray<int> d_flag;
  const char* oom = "JacobiSvd: insufficient device memory";
  if (d_sched.alloc(sched.size(), oom) || d_partial.alloc(static_cast<uint64_t>(half) * chunks * 3, oom) || d_norms.alloc(q, oom) || d_perm.alloc(q, oom) || d_flag.alloc(1, oom)) {
    *err = oom;
    return 1;
  }
  if (cudaMemcpyAsync(d_sched, sched.data(), sched.size() * sizeof(int2), cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return 1;
  const double tol = std::max(1e-15, 4.4408920985006262e-16 * sqrt(static_cast<double>(rows)));
  uint32_t sweep = 0;
  bool converged = (q == 1);
  for (; sweep < 60 && !converged; ++sweep) {
    if (cudaMemsetAsync(d_flag, 0, 4, c->stream) != cudaSuccess) break;
    for (uint32_t r = 0; r < rounds; ++r) {
      const int2* pr = d_sched + static_cast<size_t>(r) * half;
      if (fused) {
        jacobi_fused_kernel<<<half, kJacobiThreads, 0, c->stream>>>(d_a, lda, rows, pr, tol, d_flag);
        c->launches++;
      } else {
        jacobi_dots_kernel<<<dim3(half, chunks), kJacobiThreads, 0, c->stream>>>(d_a, lda, rows, pr, chunk_rows, d_partial);
        jacobi_rotate_kernel<<<dim3(half, chunks), kJacobiThreads, 0, c->stream>>>(d_a, lda, rows, pr, chunk_rows, d_partial, tol, d_flag);
        c->launches += 2;
      }
    }
    int flag = 1;
    if (cudaMemcpyAsync(&flag, d_flag, 4, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
      *err = "JacobiSvd: kernel failure";
      return 1;
    }
    converged = (flag == 0);
  }
  if (!converged) {
    *err = "JacobiSvd: no convergence in 60 sweeps (non-finite input?)";
    return 1;
  }
  if (sweeps_out) *sweeps_out = sweep;
  jacobi_colnorm_kernel<<<q, kJacobiThreads, 0, c->stream>>>(d_a, lda, rows, d_norms);
  c->launches++;
  std::vector<double> norms(q);
  if (cudaMemcpyAsync(norms.data(), d_norms, 8ull * q, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
    *err = "JacobiSvd: kernel failure";
    return 1;
  }
  std::vector<uint32_t> perm(q);
  std::iota(perm.begin(), perm.end(), 0u);
  std::stable_sort(perm.begin(), perm.end(), [&](uint32_t x, uint32_t y) { return norms[x] > norms[y]; });
  bool finite = true;
  for (uint32_t i = 0; i < out_cols; ++i) {
    sigma_host[i] = norms[perm[i]];
    finite = finite && std::isfinite(sigma_host[i]);
  }
  if (!finite) {
    *err = "JacobiSvd: non-finite singular values";
    return 1;
  }
  if (d_u && out_cols) {
    if (cudaMemcpyAsync(d_perm, perm.data(), 4ull * q, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return 1;
    jacobi_gather_kernel<<<dim3(DivUpU32(rows, 256), out_cols), 256, 0, c->stream>>>(d_a, lda, rows, d_perm, d_norms, d_u, ldu);
    c->launches++;
    if (cudaStreamSynchronize(c->stream) != cudaSuccess) {
      *err = "JacobiSvd: kernel failure";
      return 1;
    }
  }
  return 0;
}

// Host driver.  d_a (rows x q, leading dimension lda) is overwritten with U Sigma (unsorted).
// sigma_host[0..out_cols) = singular values in descending order; d_u (may be nullptr) receives the
// matching unit left singular vectors as a rows x out_cols column-major matrix (ldu).
// Returns 0, or 1 with *err set (CUDA failure / no convergence).
static int JacobiSvd(Ctx* c, double* d_a, uint64_t lda, uint32_t rows, uint32_t q, uint32_t out_cols, double* sigma_host, double* d_u, uint64_t ldu, uint32_t* sweeps_out, const char** err) {
  *err = nullptr;
  if (!q || rows < q || out_cols > q) {
    *err = "JacobiSvd: bad shape";
    return 1;
  }
  const int rc = JacobiSvdRun(c, d_a, lda, rows, q, out_cols, sigma_host, d_u, ldu, sweeps_out, err);
  if (rc && !*err) *err = "JacobiSvd: CUDA failure";
  cudaGetLastError();
  return rc;
}

}  // namespace pl2
