"""GPU parity for `--score`: the device accumulation (pl2gpu_score_*) against the numpy restatement of ScoreReport
(oracle.score_report, pinned to reference-written .sscore files in test_oracle_golden.py), and the command-line
face against those files."""
import os
import subprocess

import numpy as np
import pytest

from oracle import plink_oracle as orc
from plink_ng_b200.host import pack_genotypes, score_sums

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
ENV = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])


def _tables(entries, ref_freq, no_mean):
    w4 = np.zeros((len(entries), 4))
    d4 = np.zeros(len(entries), dtype=np.uint8)
    for k, (v, aidx, coef) in enumerate(entries):
        d0, d2 = (0, 2) if aidx else (2, 0)
        f = (1.0 - ref_freq[v]) if aidx else ref_freq[v]
        w4[k] = [coef * d0, coef, coef * d2, 0.0 if no_mean else coef * (2.0 * f)]
        d4[k] = d0 | (1 << 2) | (d2 << 4)
    return w4, d4


@pytest.mark.parametrize("n,m,no_mean", [(257, 900, False), (1000, 40000, True), (5000, 3000, False)])
def test_score_accumulation_matches_oracle(gpu_ctx, n, m, no_mean):
    """Several staging batches (16,384 entries each), several variant chunks per launch, ragged sample counts."""
    rng = np.random.default_rng(n + m)
    geno = rng.choice(4, size=(m, n), p=[0.45, 0.35, 0.17, 0.03]).astype(np.uint8)
    ref_freq = orc.ref_allele_freqs(geno)
    entries = [(int(v), int(rng.integers(0, 2)), float(rng.normal())) for v in rng.permutation(m)[: (m * 3) // 4]]
    entries.sort()
    want_nallele, _, want_dos, want_sum, _ = orc.score_report(geno, entries, ref_freq, no_mean_imputation=no_mean)
    w4, d4 = _tables(entries, ref_freq, no_mean)
    rows = pack_genotypes(geno)[[e[0] for e in entries]]
    sums, dos, miss = score_sums(gpu_ctx, rows, n, w4, d4)
    assert np.array_equal(dos.astype(np.int64), want_dos)
    assert np.array_equal(2 * len(entries) - 2 * miss.astype(np.int64), want_nallele)
    assert np.allclose(sums, want_sum, rtol=1e-11, atol=1e-11 * np.abs(want_sum).max())
    again, _, _ = score_sums(gpu_ctx, rows, n, w4, d4)
    assert np.array_equal(sums, again)  # fixed-order partial sums: bit-reproducible


def _table(path):
    rows = [ln.rstrip("\n").split("\t") for ln in open(path)]
    return rows[0], rows[1:]


@pytest.mark.parametrize("flags,golden", [(("header",), "a_sc.sscore"), (("header", "no-mean-imputation", "cols=+scoresums,+denom"), "a_sc2.sscore"),
                                          (("header", "center", "cols=+scoresums"), "a_sc_center.sscore"), (("header", "variance-standardize", "cols=+scoresums"), "a_sc_varstd.sscore"),
                                          (("header", "dominant", "list-variants", "cols=+scoresums,+denom"), "a_sc_dominant.sscore"), (("header", "recessive", "cols=+scoresums,+denom"), "a_sc_recessive.sscore")])
def test_score_cli_matches_reference_report(golden_dir, tmp_path, flags, golden):
    out = str(tmp_path / "s")
    r = subprocess.run([BIN, "--bfile", os.path.join(golden_dir, "a"), "--score", os.path.join(golden_dir, "a_score.txt"), *flags, "--out", out], capture_output=True, text=True, env=ENV)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "400 variants processed" in r.stdout and "5 entries" in r.stdout and "7 were skipped due to mismatching allele codes" in r.stdout
    got_h, got = _table(out + ".sscore")
    ref_h, ref = _table(os.path.join(golden_dir, golden))
    assert got_h == ref_h and len(got) == len(ref)
    is_float = [h.endswith("_AVG") or h.endswith("_SUM") for h in ref_h]
    same_text = 0
    for g, w in zip(got, ref):
        for col, fl in enumerate(is_float):
            if not fl:
                assert g[col] == w[col]  # IDs, phenotype, ALLELE_CT, DENOM, NAMED_ALLELE_DOSAGE_SUM: exact
            else:
                assert np.isclose(float(g[col]), float(w[col]), rtol=2e-5, atol=2e-9)  # 6 significant digits printed
                same_text += g[col] == w[col]
    assert same_text >= 0.97 * len(ref) * sum(is_float)  # fp64 sums in a different order: a last printed digit may move
    if "list-variants" in flags:
        assert open(out + ".sscore.vars", "rb").read() == open(os.path.join(golden_dir, "a_sc.sscore.vars"), "rb").read()


def test_score_header_read_names_the_column(golden_dir, tmp_path):
    out = str(tmp_path / "s")
    r = subprocess.run([BIN, "--pgen", os.path.join(golden_dir, "a_mode02.pgen"), "--pvar", os.path.join(golden_dir, "a.pvar"), "--psam", os.path.join(golden_dir, "a.psam"), "--score", os.path.join(golden_dir, "a_score.txt"), "header-read",
                        "--out", out], capture_output=True, text=True, env=ENV)
    assert r.returncode == 0, r.stdout + r.stderr
    got_h, got = _table(out + ".sscore")
    assert got_h == ["#IID", "PHENO1", "ALLELE_CT", "NAMED_ALLELE_DOSAGE_SUM", "BETA_AVG"]
    _, ref = _table(os.path.join(golden_dir, "a_sc.sscore"))
    assert [g[0:4] for g in got] == [w[1:5] for w in ref]


@pytest.mark.parametrize("n,m,cols", [(300, 1000, 3), (2000, 5000, 50)])
def test_variant_scores_match_oracle(gpu_ctx, n, m, cols):
    """--variant-score on the approx-PCA tile path: several 128-variant CTAs, a second column group (50 > 32 columns),
    monomorphic variants (centred dosage 0 -> the 2 f W term alone), samples with weight 0."""
    from plink_ng_b200.host import variant_scores

    rng = np.random.default_rng(n + cols)
    geno = rng.choice(4, size=(m, n), p=[0.5, 0.3, 0.17, 0.03]).astype(np.uint8)
    geno[5] = 0
    geno[6] = np.where(rng.random(n) < 0.1, 3, 2)
    w = rng.normal(size=(n, cols))
    w[rng.random(n) < 0.2] = 0.0
    want = orc.variant_scores(geno, w, orc.ref_allele_freqs(geno))
    got = variant_scores(gpu_ctx, pack_genotypes(geno), n, w)
    assert np.allclose(got, want, rtol=1e-10, atol=1e-9 * np.abs(want).max())


@pytest.mark.parametrize("flags,golden", [((), "a_vs.vscore"), (("cols=+altfreq",), "a_vs_altfreq.vscore")])
def test_variant_score_cli_matches_reference_report(golden_dir, tmp_path, flags, golden):
    out = str(tmp_path / "v")
    r = subprocess.run([BIN, "--bfile", os.path.join(golden_dir, "a"), "--variant-score", os.path.join(golden_dir, "a_vscore_weights.txt"), *flags, "--out", out], capture_output=True, text=True, env=ENV)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "2 score-vectors loaded for 89 samples" in r.stdout and "1 line skipped" in r.stdout
    got_h, got = _table(out + ".vscore")
    ref_h, ref = _table(os.path.join(golden_dir, golden))
    assert got_h == ref_h and len(got) == len(ref)
    first_score = ref_h.index("W1")
    same_text = 0
    for g, w in zip(got, ref):
        assert g[:first_score] == w[:first_score]  # CHROM POS ID REF ALT PROVISIONAL_REF? [ALT_FREQ]: exact
        for col in range(first_score, len(ref_h)):
            assert np.isclose(float(g[col]), float(w[col]), rtol=2e-5, atol=2e-9)
            same_text += g[col] == w[col]
    assert same_text >= 0.97 * len(ref) * (len(ref_h) - first_score)
