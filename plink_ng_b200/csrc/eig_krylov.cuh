// eig_krylov.cuh - leading eigenpairs of a resident dense symmetric matrix by restarted block Krylov iteration with
// Rayleigh-Ritz extraction: the scalable replacement for dsyevr in the exact `--pca` branch (CalcPca :5942-6040 ->
// ExtractEigvecs, 2.0/plink2_matrix.cc:1089) once the sample count makes an O(N^3) dense factorization the wrong tool.
//
// One restart:  K = [X, AX, ..., A^p X]  (N x b(p+1), b = k + 8 guard vectors, p = 5)
//               Q  = orthonormal basis of K: block Gram-Schmidt, three projection passes per block, each followed by a
//                    one-sided Jacobi SVD of the N x b residual (the construction pca.cu uses for the approx branch)
//               T  = Q^T (A Q), eigenpairs of T by Jacobi  ->  X = Q V_b  (the b leading Ritz vectors)
//               stop when  || A x_i - theta_i x_i ||  <=  tol * theta_1  for the k wanted pairs.
// Every product is a dense_fp64.cuh GEMM (fixed-order split sums), so a run is bit-reproducible.  Cost per restart
// (2p + 1) b N^2 MACs, all HBM/L2-resident: 0.3 s at N = 46,340, where one Jacobi sweep over the matrix costs minutes.
#pragma once
#include <random>

#include "common.cuh"
#include "dense_fp64.cuh"
#include "jacobi.cuh"

namespace pl2 {

// per column i < cols: out[2 i] = x_i . (A x)_i (Rayleigh quotient of a unit x_i), out[2 i + 1] = || (A x)_i - out[2 i] x_i ||^2
static __global__ void __launch_bounds__(256) ritz_residual_kernel(const double* __restrict__ x, const double* __restrict__ ax, uint64_t ld, uint32_t rows, double* __restrict__ out) {
  __shared__ double red[8];
  const double* xc = x + static_cast<uint64_t>(blockIdx.x) * ld;
  const double* ac = ax + static_cast<uint64_t>(blockIdx.x) * ld;
  double rq = 0.0;
  for (uint32_t r = threadIdx.x; r < rows; r += 256) rq = fma(xc[r], ac[r], rq);
#pragma unroll
  for (int o = 16; o; o >>= 1) rq += __shfl_xor_sync(0xFFFFFFFFu, rq, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = rq;
  __syncthreads();
  double theta = 0.0;
  for (int i = 0; i < 8; ++i) theta += red[i];
  __syncthreads();
  double rs = 0.0;
  for (uint32_t r = threadIdx.x; r < rows; r += 256) {
    const double d = ac[r] - theta * xc[r];
    rs = fma(d, d, rs);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) rs += __shfl_xor_sync(0xFFFFFFFFu, rs, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = rs;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < 8; ++i) tot += red[i];
    out[2 * blockIdx.x] = theta;
    out[2 * blockIdx.x + 1] = tot;
  }
}

// Orthonormalises the block_ct blocks of block_cols columns of q (rows x block_ct block_cols, leading dimension ld) in
// place, block by block.  d_c: >= (block_ct block_cols) x block_cols doubles; d_cpart: DgemmTN partial buffer for the
// widest projection; d_tmp: rows x block_cols.
static int BlockOrthonormalize(Ctx* c, double* q, uint64_t ld, uint32_t rows, uint32_t block_cols, uint32_t block_ct, double* d_c, double* d_cpart, double* d_tmp, const char** err) {
  std::vector<double> sig(block_cols);
  for (uint32_t t = 0; t < block_ct; ++t) {
    double* w = q + static_cast<uint64_t>(t) * block_cols * ld;
    const uint32_t prev = t * block_cols;
    for (int rep = 0; rep < 3; ++rep) {
      if (prev && (DgemmTN(c, q, ld, prev, w, ld, block_cols, rows, d_cpart, d_c, prev) || DgemmNN(c, q, ld, rows, prev, d_c, prev, block_cols, w, ld, true, nullptr))) return 1;
      if (JacobiSvd(c, w, ld, rows, block_cols, block_cols, sig.data(), d_tmp, rows, nullptr, err)) return 1;
      if (cudaMemcpy2DAsync(w, ld * 8, d_tmp, static_cast<uint64_t>(rows) * 8, static_cast<uint64_t>(rows) * 8, block_cols, cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess) return 1;
    }
  }
  return 0;
}

// SymEigTopKKrylov after its size check, with b columns per block and p Krylov steps: the scratch is freed on return,
// before SymEigTopKKrylov clears the CUDA error state
static int SymEigTopKKrylovRun(Ctx* c, const double* d_a, uint32_t n, uint32_t k, uint32_t b, uint32_t p, double* eigvals_host, double* d_u, uint32_t* restarts_out, const char** err) {
  const uint32_t q = b * (p + 1);
  DevArray<double> d_q, d_aq, d_t, d_tu, d_x, d_ax, d_c, d_cpart, d_tmp, d_res;
  uint64_t part = DgemmTNPartialDoubles(c, q, q, n);
  for (uint32_t t = 1; t <= p; ++t) part = std::max(part, DgemmTNPartialDoubles(c, t * b, b, n));
  const uint64_t nq = static_cast<uint64_t>(n) * q, nb = static_cast<uint64_t>(n) * b;
  const char* oom = "insufficient device memory for the Krylov basis";
  if (d_q.alloc(nq, oom) || d_aq.alloc(nq, oom) || d_t.alloc(1ull * q * q, oom) || d_tu.alloc(1ull * q * b, oom) || d_x.alloc(nb, oom) || d_ax.alloc(nb, oom) || d_c.alloc(1ull * q * b, oom) || d_cpart.alloc(part, oom) ||
      d_tmp.alloc(nb, oom) || d_res.alloc(2ull * b, oom)) {
    *err = oom;
    return 1;
  }
  {  // deterministic Gaussian start block
    std::vector<double> x0(nb);
    std::mt19937_64 gen(20260923);
    std::normal_distribution<double> nd(0.0, 1.0);
    for (double& v : x0) v = nd(gen);
    if (cudaMemcpyAsync(d_x, x0.data(), nb * 8, cudaMemcpyHostToDevice, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) return 1;
  }
  std::vector<double> theta(q), res(2ull * b);
  const double tol = 1e-10;
  uint32_t it = 0;
  bool converged = false, failed = false;
  for (; it < 400 && !converged; ++it) {
    // Krylov blocks
    if (cudaMemcpyAsync(d_q, d_x, nb * 8, cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess) { failed = true; break; }
    for (uint32_t j = 1; j <= p && !failed; ++j) failed = DgemmNN(c, d_a, n, n, n, d_q + static_cast<uint64_t>(j - 1) * nb, n, b, d_q + static_cast<uint64_t>(j) * nb, n, false, nullptr) != 0;
    if (failed) break;
    if (BlockOrthonormalize(c, d_q, n, n, b, p + 1, d_c, d_cpart, d_tmp, err)) { failed = true; break; }
    // Rayleigh-Ritz
    if (DgemmNN(c, d_a, n, n, n, d_q, n, q, d_aq, n, false, nullptr) || DgemmTN(c, d_q, n, q, d_aq, n, q, n, d_cpart, d_t, q)) { failed = true; break; }
    if (JacobiSvd(c, d_t, q, q, q, b, theta.data(), d_tu, q, nullptr, err)) { failed = true; break; }
    if (DgemmNN(c, d_q, n, n, q, d_tu, q, b, d_x, n, false, nullptr) || DgemmNN(c, d_aq, n, n, q, d_tu, q, b, d_ax, n, false, nullptr)) { failed = true; break; }
    ritz_residual_kernel<<<b, 256, 0, c->stream>>>(d_x, d_ax, n, n, d_res);
    c->launches++;
    if (cudaMemcpyAsync(res.data(), d_res, 16ull * b, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) { failed = true; break; }
    double worst = 0.0;
    for (uint32_t i = 0; i < k; ++i) worst = std::max(worst, sqrt(res[2 * i + 1]));
    converged = worst <= tol * fabs(res[0]);
  }
  if (failed) {
    if (!*err) *err = "CUDA failure in the Krylov solver";
    return 1;
  }
  if (!converged) {
    *err = "Krylov eigensolver did not converge in 400 restarts";
    return 1;
  }
  // the Ritz values came out as singular values of T (|theta|); the Rayleigh quotients carry the sign
  bool ordered = true;
  for (uint32_t i = 0; i < k; ++i) {
    eigvals_host[i] = res[2 * i];
    ordered = ordered && res[2 * i] > 0.0 && (i == 0 || res[2 * i] <= res[2 * (i - 1)] * (1 + 1e-12));
  }
  if (!ordered) {
    *err = "leading eigenvalues are not positive and descending (indefinite matrix?)";
    return 1;
  }
  if (cudaMemcpyAsync(d_u, d_x, static_cast<uint64_t>(n) * k * 8, cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
    *err = "CUDA failure in the Krylov solver";
    return 1;
  }
  if (restarts_out) *restarts_out = it;
  return 0;
}

// d_a: symmetric n x n (column-major == row-major), untouched.  eigvals_host[k] descending, d_u: n x k unit eigenvectors
// (leading dimension n).  Returns 0, or 1 with *err set.
static int SymEigTopKKrylov(Ctx* c, const double* d_a, uint32_t n, uint32_t k, double* eigvals_host, double* d_u, uint32_t* restarts_out, const char** err) {
  *err = nullptr;
  const uint32_t b = std::min(n, k + 8);
  uint32_t p = 5;
  while (p > 1 && static_cast<uint64_t>(b) * (p + 1) > n) --p;
  if (static_cast<uint64_t>(b) * (p + 1) > n) {
    *err = "matrix too small for the Krylov solver";
    return 1;
  }
  const int rc = SymEigTopKKrylovRun(c, d_a, n, k, b, p, eigvals_host, d_u, restarts_out, err);
  cudaGetLastError();
  return rc;
}

}  // namespace pl2
