"""GPU parity: exact --pca (top-k eigenpairs of the GPU-built GRM) vs numpy eigh of the oracle GRM
and vs the reference's .eigenval/.eigenvec (LAPACK-enabled oracle build), sign-flip tolerant like
the reference's own comparer (2.0/Tests/TEST_PHASED_VCF/pca_compare.py:75-80)."""
import os
import subprocess

import numpy as np
import pytest

from plink_ng_b200.host import GrmJob, pack_genotypes
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")


def _structured_geno(m, n, seed, pops=4, fst=0.08, miss=0.01):
    """Balding-Nichols populations so the leading eigenvalues are well separated (SURVEY 8c caveat)."""
    rng = np.random.default_rng(seed)
    anc = rng.uniform(0.1, 0.9, size=m)
    a = anc * (1 - fst) / fst
    b = (1 - anc) * (1 - fst) / fst
    pf = rng.beta(a[:, None], b[:, None], size=(m, pops))
    lab = rng.integers(0, pops, size=n)
    f = pf[:, lab]
    g = (rng.random((m, n)) < f).astype(np.uint8) + (rng.random((m, n)) < f).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


def _align(vecs, ref):
    s = np.sign(np.sum(vecs * ref, axis=1, keepdims=True))
    s[s == 0] = 1
    return vecs * s


def test_exact_pca_matches_numpy_eigh(gpu_ctx):
    n, m, k = 300, 4000, 5
    geno = _structured_geno(m, n, seed=4)
    want, _ = orc.grm(geno)
    w, v = np.linalg.eigh(want)
    w, v = w[::-1][:k], v[:, ::-1][:, :k].T
    with GrmJob(gpu_ctx, n) as job:
        job.add_variants(pack_genotypes(geno))
        vals, vecs = job.eigen_topk(k)
    assert np.allclose(vals, w, rtol=1e-8)
    assert np.allclose(_align(vecs[:3], v[:3]), v[:3], atol=1e-5 * np.abs(v[:3]).max())  # 3 structure PCs: 1e-5 relative
    assert np.allclose(np.linalg.norm(vecs, axis=1), 1.0, atol=1e-12)


@pytest.mark.parametrize("n,m,k,force", [(1200, 6000, 8, True), (4500, 7000, 6, False)])
def test_exact_pca_block_krylov_matches_numpy_eigh(gpu_ctx, monkeypatch, n, m, k, force):
    """Exact --pca beyond Jacobi's reach: restarted block Krylov + Rayleigh-Ritz on the resident GRM (eig_krylov.cuh),
    the default above 4,096 samples (forced through PL2_EIGEN at the small size).  Structure and noise-level
    eigenvalues alike must agree with LAPACK's to 1e-8: this solver converges every wanted pair to a 1e-10 residual."""
    if force:
        monkeypatch.setenv("PL2_EIGEN", "krylov")
    geno = _structured_geno(m, n, seed=n, pops=5, fst=0.08)
    want, _ = orc.grm(geno)
    w, v = np.linalg.eigh(want)
    w, v = w[::-1][:k], v[:, ::-1][:, :k].T
    with GrmJob(gpu_ctx, n) as job:
        job.add_variants(pack_genotypes(geno))
        vals, vecs = job.eigen_topk(k)
    assert np.allclose(vals, w, rtol=1e-8)
    assert np.allclose(_align(vecs[:4], v[:4]), v[:4], atol=1e-6 * np.abs(v[:4]).max())  # 4 structure PCs
    assert np.allclose(np.linalg.norm(vecs, axis=1), 1.0, atol=1e-10)
    # noise-level eigenvectors: compare the invariant subspace residual instead of ill-conditioned individual vectors
    resid = want @ vecs.T - vecs.T * vals
    assert np.abs(resid).max() < 1e-7 * vals[0]


def test_exact_pca_cli_matches_reference_files(golden_dir, tmp_path):
    out = str(tmp_path / "p")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    r = subprocess.run([BIN, "--bfile", os.path.join(golden_dir, "a"), "--pca", "4", "--out", out], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    ref_val = np.loadtxt(os.path.join(golden_dir, "a_pca.eigenval"))
    got_val = np.loadtxt(out + ".eigenval")
    assert np.allclose(got_val, ref_val, rtol=3e-6)
    ref = [ln.rstrip("\n").split("\t") for ln in open(os.path.join(golden_dir, "a_pca.eigenvec"))]
    got = [ln.rstrip("\n").split("\t") for ln in open(out + ".eigenvec")]
    assert got[0] == ref[0] and [g[:2] for g in got] == [g[:2] for g in ref]
    rv = np.array([x[2:] for x in ref[1:]], dtype=float).T
    gv = np.array([x[2:] for x in got[1:]], dtype=float).T
    # unstructured --dummy data: eigenvalue gaps ~1e-2, so eigenvectors are compared at the
    # 6-significant-digit print precision amplified by 1/gap
    assert np.allclose(_align(gv, rv), rv, atol=2e-4)


@pytest.mark.parametrize("algo", ["tensor", "fp64"])
def test_approx_pca_matches_oracle_same_gaussian_start(gpu_ctx, algo, monkeypatch):
    """Both pass implementations: the int8 tensor path (pca_ts_kernels.cuh, dense factor in 32-bit fixed point) and the
    CUDA-core fp64 kernels (pca_kernels.cuh) kept as a cross-check."""
    from plink_ng_b200.host import pca_approx

    monkeypatch.setenv("PL2_PCA_ALGO", algo)
    n, m, k = 400, 6000, 5  # 2k = 10 columns: a column group padded to 12; q = 60 -> groups of 48 + 12
    geno = _structured_geno(m, n, seed=9, pops=6, fst=0.1)
    g1 = np.random.default_rng(1).standard_normal((n, 2 * k))
    want_vals, want_vecs = orc.pca_approx(geno, k, g1)
    vals, vecs = pca_approx(gpu_ctx, pack_genotypes(geno), n, k, g1)
    assert np.allclose(vals, want_vals, rtol=1e-6)
    # 6 populations -> 5 structure PCs with well separated eigenvalues: north_star's 1e-5 (relative to the
    # largest component) applies
    assert np.allclose(_align(vecs, want_vecs), want_vecs, atol=1e-5 * np.abs(want_vecs).max())
    # and the approximation is a good one: close to the exact eigenpairs of the mean-imputed GRM
    g, _ = orc.grm(geno, meanimpute=True)
    ev, _ = orc.pca_exact(g, k)
    assert np.allclose(vals, ev, rtol=2e-2)


def test_approx_pca_k20_tensor_path_matches_oracle(gpu_ctx):
    """BASELINE's --pca 20 shape at a size numpy finishes in seconds: 40-column passes (one column group of N = 160),
    840-column final projection (17 groups of 48 + one of 24), several 128-variant / 256-sample tiles and split-K."""
    from plink_ng_b200.host import pca_approx

    n, m, k = 1100, 9000, 20
    geno = _structured_geno(m, n, seed=21, pops=8, fst=0.12)
    g1 = np.random.default_rng(3).standard_normal((n, 2 * k))
    want_vals, want_vecs = orc.pca_approx(geno, k, g1)
    vals, vecs = pca_approx(gpu_ctx, pack_genotypes(geno), n, k, g1)
    top = 7  # 8 populations -> 7 structure PCs
    assert np.allclose(vals[:top], want_vals[:top], rtol=1e-9)
    assert np.allclose(_align(vecs[:top], want_vecs[:top]), want_vecs[:top], atol=1e-5 * np.abs(want_vecs[:top]).max())
    # The 13 noise-level eigenvalues are Ritz values over a numerically rank-deficient Krylov space (its singular
    # values span 1e35 .. 1e-4): LAPACK's SVD in the restatement, one-sided Jacobi and block Gram-Schmidt each complete
    # the basis differently there, and the values move by 1e-4 .. 1e-3 (tests/harness/pca_basis_compare.py; the
    # reference's own comparison against PLINK 1.9 allows 9e-3, 2.0/Tests/TEST_PHASED_VCF/run_tests.sh:76-99).
    assert np.allclose(vals[top:], want_vals[top:], rtol=3e-3)


@pytest.mark.parametrize("basis,final", [("jacobi", "jacobi"), ("jacobi", "gram"), ("bcgs", "jacobi")])
def test_approx_pca_alternative_factorizations_agree(gpu_ctx, monkeypatch, basis, final):
    """The non-default ways through the two dense factorizations (PL2_PCA_BASIS / PL2_PCA_FINAL) give the same
    structure PCs as the default (block Gram-Schmidt basis, Gram-matrix final stage)."""
    from plink_ng_b200.host import pca_approx

    n, m, k = 700, 5000, 8
    geno = _structured_geno(m, n, seed=33, pops=6, fst=0.1)
    g1 = np.random.default_rng(5).standard_normal((n, 2 * k))
    ref_vals, ref_vecs = pca_approx(gpu_ctx, pack_genotypes(geno), n, k, g1)
    monkeypatch.setenv("PL2_PCA_BASIS", basis)
    monkeypatch.setenv("PL2_PCA_FINAL", final)
    vals, vecs = pca_approx(gpu_ctx, pack_genotypes(geno), n, k, g1)
    assert np.allclose(vals[:5], ref_vals[:5], rtol=1e-9) and np.allclose(vals, ref_vals, rtol=3e-3)
    assert np.allclose(_align(vecs[:5], ref_vecs[:5]), ref_vecs[:5], atol=1e-6 * np.abs(ref_vecs[:5]).max())


def test_approx_pca_cli_matches_reference_files(golden_dir, tmp_path):
    """Same --seed => same SFMT/Box-Muller start matrix as the reference run that wrote the golden files."""
    out = str(tmp_path / "pa")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    r = subprocess.run([BIN, "--bfile", os.path.join(golden_dir, "a"), "--pca", "3", "approx", "--seed", "11", "--threads", "2", "--out", out], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    ref_val = np.loadtxt(os.path.join(golden_dir, "a_pcaa.eigenval"))
    got_val = np.loadtxt(out + ".eigenval")
    assert np.allclose(got_val, ref_val, rtol=1e-5)
    ref = [ln.rstrip("\n").split("\t") for ln in open(os.path.join(golden_dir, "a_pcaa.eigenvec"))]
    got = [ln.rstrip("\n").split("\t") for ln in open(out + ".eigenvec")]
    assert got[0] == ref[0]
    rv = np.array([x[2:] for x in ref[1:]], dtype=float).T
    gv = np.array([x[2:] for x in got[1:]], dtype=float).T
    # unstructured 100-sample data: near-degenerate eigenvalues amplify last-digit differences
    assert np.allclose(_align(gv, rv), rv, atol=5e-4)
