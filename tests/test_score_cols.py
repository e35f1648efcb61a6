"""CPU: several `--score` coefficient columns in one pass (--score-col-nums) and weight-column selection for
`--variant-score` (--vscore-col-nums).

A numpy restatement of ScoreReport for several columns is pinned to the reference's reports on set A
(tests/golden/make_score_cols_set.py); the command-line parsing and its errors are checked on the host program; and
the host driver is replayed on the CPU through the stand-in libraries (tests/harness/mock_score_cols.cc ahead of
tests/harness/mock_pl2gpu.cc, injected with LD_PRELOAD as in test_host_orchestration.py), whose reports must match the
reference's to the printed digits.  The goldens are stored gzipped."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from oracle import plink_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")


# ------------------------------------------------------------------------------- numpy restatement
def score_file_entries_cols(path, ids, ref_alleles, alt_alleles, cols, header=True, id_col=0, allele_col=1):
    """The (variant index, named-allele index 0 = REF / 1 = ALT, coefficient vector) triples ScoreReport keeps, in file
    order (2.0/plink2_matrix_calc.cc:7712-7790), for the 0-based coefficient token indices `cols` (increasing, as
    --score-col-nums selects them)."""
    idx = {v: k for k, v in enumerate(ids)}
    out, missing_id, missing_allele = [], 0, 0
    with gzip.open(path, "rt") as f:
        if header:
            f.readline()
        for ln in f:
            t = ln.split()
            if not t:
                continue
            k = idx.get(t[id_col])
            if k is None:
                missing_id += 1
                continue
            a = t[allele_col]
            if a not in (ref_alleles[k], alt_alleles[k]):
                missing_allele += 1
                continue
            out.append((k, 0 if a == ref_alleles[k] else 1, np.array([float(t[c]) for c in cols])))
    return out, missing_id, missing_allele


def score_report_cols(geno, entries, ref_freq, no_mean_imputation=False, mode=""):
    """oracle.score_report for several coefficient columns (2.0/plink2_matrix_calc.cc:7186-7234, report :8520-8539).
    The per-variant dosage table (slope, intercept, missing dosage, with the reference's uncentred missing-call term)
    does not depend on the column; each column scales it by its own coefficient.  Missing calls, and so ALLELE_CT and
    DENOM, count once per variant when a file names both of its alleles (:7788).  Returns ALLELE_CT, DENOM,
    NAMED_ALLELE_DOSAGE_SUM per sample, and the sums and averages as [sample, column]."""
    n = geno.shape[1]
    ssum = np.zeros((n, len(entries[0][2])))
    dos = np.zeros(n, dtype=np.int64)
    for v, aidx, coefs in entries:
        g = geno[v]
        named = np.where(g == 3, 0, g if aidx == 1 else 2 - g).astype(np.int64)
        f_named = (1.0 - ref_freq[v]) if aidx == 1 else ref_freq[v]
        slope, icpt = 1.0, 0.0
        if mode in ("center", "variance-standardize"):
            if mode == "variance-standardize":
                var = 2.0 * f_named * (1.0 - f_named)
                slope = 1.0 / np.sqrt(var) if var > orc.SMALL_EPSILON else 0.0
            icpt = (-2.0 * f_named) * slope
        miss_dosage = 2.0 * f_named
        if mode in ("dominant", "recessive"):
            named = np.minimum(named, 1) if mode == "dominant" else np.maximum(named - 1, 0)
            miss_dosage = f_named
        d = named.astype(np.float64) * slope + icpt
        d = np.where(g == 3, 0.0 if no_mean_imputation else miss_dosage * slope, d)
        ssum += d[:, None] * coefs[None, :]
        dos += named
    variants = sorted({e[0] for e in entries})
    miss = (geno[variants] == 3).sum(axis=0)
    denom_full = 2 * len(variants)
    nallele = denom_full - 2 * miss
    denom = nallele if no_mean_imputation else np.full(n, denom_full)
    return nallele, denom, dos, ssum, ssum * (1.0 / denom)[:, None]


# golden -> (score file, header line present, 0-based ID / allele / coefficient tokens, names, flags, restatement mode)
NAMES = ["BETA", "NEG", "ZERO", "MIX", "HALF"]
CASES = {
    "a_scc.sscore": ("a_score_cols.txt.gz", False, 0, 1, [2, 3, 4, 5, 6], ["SCORE1", "SCORE2", "SCORE3", "SCORE4", "SCORE5"], ["--score", "a_score_cols.txt.gz", "--score-col-nums", "3-7"], False, ""),
    "a_scc_hr.sscore": ("a_score_cols.txt.gz", True, 0, 1, [2, 3, 4, 5, 6], NAMES, ["--score", "a_score_cols.txt.gz", "header-read", "--score-col-nums", "3-7"], False, ""),
    "a_scc_nmi.sscore": ("a_score_cols.txt.gz", True, 0, 1, [2, 3, 4, 5, 6], NAMES, ["--score", "a_score_cols.txt.gz", "header-read", "no-mean-imputation", "cols=+scoresums,+denom", "--score-col-nums", "3-7"], True, ""),
    "a_scc_vs.sscore": ("a_score_cols.txt.gz", True, 0, 1, [2, 3, 4, 5, 6], NAMES, ["--score", "a_score_cols.txt.gz", "header-read", "variance-standardize", "cols=+scoresums", "--score-col-nums", "3-7"], False, "variance-standardize"),
    "a_scc_dom.sscore": ("a_score_cols.txt.gz", True, 0, 1, [2, 3, 4, 5, 6], NAMES, ["--score", "a_score_cols.txt.gz", "header-read", "dominant", "cols=+scoresums", "--score-col-nums", "3-7"], False, "dominant"),
    "a_scc_ord.sscore": ("a_score_cols.txt.gz", True, 0, 1, [2, 4, 5, 6], ["BETA", "ZERO", "MIX", "HALF"], ["--score", "a_score_cols.txt.gz", "header-read", "cols=+scoresums", "--score-col-nums", "6", "5-7,3"], False, ""),
    "a_scc_pc.sscore": ("a_pcw.eigenvec.allele.gz", True, 1, 5, list(range(6, 16)), ["PC%d" % k for k in range(1, 11)],
                        ["--score", "a_pcw.eigenvec.allele.gz", "2", "6", "header-read", "no-mean-imputation", "variance-standardize", "--score-col-nums", "7-16", "--read-freq", "a_pcw.afreq.gz"], True, "variance-standardize"),
}


def _text(path):
    """A golden (gzipped) or an output (plain) as text."""
    return (gzip.open(path, "rt") if path.endswith(".gz") else open(path)).read()


def _table(path):
    rows = [ln.split("\t") for ln in _text(path).rstrip("\n").split("\n")]
    return rows[0], np.array(rows[1:])


def _set_a():
    geno = orc.read_bed(os.path.join(GD, "a.bed"), 100)
    bim = [ln.split() for ln in open(os.path.join(GD, "a.bim"))]
    return geno, [b[1] for b in bim], [b[5] for b in bim], [b[4] for b in bim]


@pytest.mark.parametrize("gold", sorted(CASES))
def test_restatement_matches_reference_reports(gold, tmp_path):
    """Integer columns exact; every _AVG / _SUM column to the 6 printed digits; names and column order as written."""
    geno, ids, ref, alt = _set_a()
    fname, header, id_col, allele_col, cols, names, args, no_mean, mode = CASES[gold]
    entries, _, _ = score_file_entries_cols(os.path.join(GD, fname), ids, ref, alt, cols, header=header, id_col=id_col, allele_col=allele_col)
    rf = orc.ref_allele_freqs(geno)
    if "--read-freq" in args:
        (tmp_path / "a_pcw.afreq").write_text(_text(os.path.join(GD, "a_pcw.afreq.gz")))
        rf = orc.read_freq_overrides(str(tmp_path / "a_pcw.afreq"), ids, ref, alt)
    nallele, denom, dos, ssum, avg = score_report_cols(geno, entries, rf, no_mean_imputation=no_mean, mode=mode)
    h, r = _table(os.path.join(GD, gold + ".gz"))
    assert [x for x in h if x.endswith("_AVG")] == [nm + "_AVG" for nm in names]
    assert np.array_equal(r[:, h.index("ALLELE_CT")].astype(int), nallele) and np.array_equal(r[:, h.index("NAMED_ALLELE_DOSAGE_SUM")].astype(int), dos)
    if "DENOM" in h:
        assert np.array_equal(r[:, h.index("DENOM")].astype(int), denom)
    for j, nm in enumerate(names):
        assert np.allclose(r[:, h.index(nm + "_AVG")].astype(float), avg[:, j], rtol=1e-5, atol=1e-9)
        if nm + "_SUM" in h:
            assert np.allclose(r[:, h.index(nm + "_SUM")].astype(float), ssum[:, j], rtol=1e-5, atol=1e-9)


def test_restatement_of_the_selected_weight_column_matches_reference():
    geno, _, _, _ = _set_a()
    iid = [ln.split()[1] for ln in open(os.path.join(GD, "a.fam"))]
    w = np.zeros((len(iid), 1))
    for ln in open(os.path.join(GD, "a_vscore_weights.txt")).read().split("\n")[1:]:
        t = ln.split("\t")
        if len(t) == 3 and t[0] in iid:
            w[iid.index(t[0]), 0] = float(t[2])
    want = orc.variant_scores(geno, w, orc.ref_allele_freqs(geno))
    h, r = _table(os.path.join(GD, "a_vsc.vscore.gz"))
    assert h[-1] == "W2" and "W1" not in h
    assert np.allclose(r[:, -1].astype(float), want[:, 0], rtol=1e-5, atol=1e-9)


# ------------------------------------------------------------------------------- command line
def _cli(args, env=None):
    return subprocess.run([BIN, "--bfile", "a"] + args + ["--out", os.path.join(os.environ.get("TMPDIR", "/tmp"), "pl2_score_cols_cli")], capture_output=True, text=True, cwd=GD, env=env)


@pytest.mark.parametrize("args,msg", [
    (["--freq", "--score-col-nums", "3"], "--score-col-nums must be used with --score[-list]."),
    (["--score", "a_score_cols.txt.gz", "1", "2", "3", "--score-col-nums", "4-5"], "--score-col-nums cannot be used when three numeric arguments are\nprovided to --score."),
    (["--score-col-nums", "4-5", "--score", "a_score_cols.txt.gz", "1", "2", "3"], "--score-col-nums cannot be used when three numeric arguments are\nprovided to --score."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "1,3"], "--score variant ID column index matches a coefficient column index."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "2-4"], "--score allele column index matches a coefficient column index."),
    (["--score", "a_score_cols.txt.gz", "2", "1", "--score-col-nums", "2-3"], "--score variant ID column index matches a coefficient column index."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "5-3"], "Invalid --score-col-nums range '5-3'."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "3-3"], "Duplicate --score-col-nums argument '3'."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "3-"], "Invalid --score-col-nums argument '3-'."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "3,x"], "Invalid --score-col-nums argument 'x'."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "0"], "Invalid --score-col-nums argument '0'."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "3-5", "5"], "Duplicate --score-col-nums argument '5'."),
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", ","], "--score-col-nums requires at least one value."),
    (["--freq", "--vscore-col-nums", "2"], "--vscore-col-nums must be used with --variant-score."),
    (["--variant-score", "a_vscore_weights.txt", "--vscore-col-nums", "2-1"], "Invalid --vscore-col-nums range '2-1'."),
])
def test_command_line_errors(args, msg):
    """The reference's wording; invalid command lines exit with code 8, before any device work."""
    r = _cli(args)
    assert r.returncode == 8, r.stdout + r.stderr
    assert "Error: " + msg in r.stdout + r.stderr


@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    """The several-column score stand-in first, so its score_* symbols are the ones the host program binds."""
    d = tmp_path_factory.mktemp("mock")
    sos = []
    for name in ("mock_score_cols", "mock_pl2gpu"):
        so = str(d / (name + ".so"))
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", name + ".cc")], check=True)
        sos.append(so)
    return " ".join(sos)


def _replay(mock_so, args, out):
    env = dict(os.environ, LD_PRELOAD=mock_so, PL2_MOCK_DEVICES="1")
    return subprocess.run([BIN, "--bfile", "a"] + args + ["--out", out], capture_output=True, text=True, env=env, cwd=GD)


@pytest.mark.parametrize("args,msg,code", [
    (["--score", "a_score_cols.txt.gz", "--score-col-nums", "3-8"], "Line 2 of --score file has fewer tokens than expected.", 6),  # line 1: an unknown ID
    (["--score", "a_score_cols.txt.gz", "header-read", "--score-col-nums", "3-8"], "Line 1 of --score file has fewer tokens than expected.", 6),
    (["--variant-score", "a_vscore_weights.txt", "--vscore-col-nums", "1-2"], "--vscore-col-nums argument overlaps with ID columns.", 7),
    (["--variant-score", "a_vscore_weights.txt", "--vscore-col-nums", "3-4"], "Line 1 of --variant-score file has fewer tokens than expected.", 7),
])
def test_file_errors_replayed_on_the_cpu(mock_so, tmp_path, args, msg, code):
    r = _replay(mock_so, args, str(tmp_path / "o"))
    assert r.returncode == code, r.stdout + r.stderr
    assert "Error: " + msg in r.stdout + r.stderr


def test_duplicate_score_names_are_refused(mock_so, tmp_path):
    path = tmp_path / "dup.txt"
    lines = _text(os.path.join(GD, "a_score_cols.txt.gz")).split("\n")
    path.write_text("\n".join([lines[0].replace("MIX", "NEG")] + lines[1:]))
    r = _replay(mock_so, ["--score", str(path), "header-read", "--score-col-nums", "3-7"], str(tmp_path / "o"))
    assert r.returncode == 6 and "Error: --score: Score IDs are not unique." in r.stdout, r.stdout
    r = _replay(mock_so, ["--score", str(path), "header-read", "--score-col-nums", "3,5"], str(tmp_path / "o"))
    assert r.returncode == 0, r.stdout  # only the selected columns need distinct names


def _text_close(path, gold, rtol=2e-5, atol=2e-9):
    got = open(path).read().split("\n")
    ref = _text(os.path.join(GD, gold + ".gz")).split("\n")
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        if a != b:
            ta, tb = a.split("\t"), b.split("\t")
            assert len(ta) == len(tb)
            for x, y in zip(ta, tb):
                assert x == y or abs(float(x) - float(y)) <= rtol * abs(float(y)) + atol, (a, b)


@pytest.mark.parametrize("gold", sorted(CASES))
def test_score_driver_replayed_on_the_cpu(mock_so, tmp_path, gold):
    out = str(tmp_path / "o")
    r = _replay(mock_so, CASES[gold][6], out)
    assert r.returncode == 0, r.stdout + r.stderr
    _text_close(out + ".sscore", gold)


def test_variant_score_column_selection_replayed_on_the_cpu(mock_so, tmp_path):
    out = str(tmp_path / "o")
    r = _replay(mock_so, ["--variant-score", "a_vscore_weights.txt", "--vscore-col-nums", "3"], out)
    assert r.returncode == 0, r.stdout + r.stderr
    _text_close(out + ".vscore", "a_vsc.vscore", atol=1e-9)


@pytest.mark.parametrize("k", [3, 5, 7])
def test_one_selected_column_is_the_three_number_form(mock_so, tmp_path, k):
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    assert _replay(mock_so, ["--score", "a_score_cols.txt.gz", "header-read", "cols=+scoresums", "--score-col-nums", str(k)], a).returncode == 0
    assert _replay(mock_so, ["--score", "a_score_cols.txt.gz", "1", "2", str(k), "header-read", "cols=+scoresums"], b).returncode == 0
    assert open(a + ".sscore", "rb").read() == open(b + ".sscore", "rb").read()
