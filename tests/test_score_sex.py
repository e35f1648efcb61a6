"""CPU: `--score` and `--variant-score` on chrX, chrY and MT with the reference's sex-dependent ploidy, and
--xchr-model.

A numpy restatement of the reference's rules is pinned to its reports on set X (tests/golden/make_score_sex_set.py):
integer columns exact (NAMED_ALLELE_DOSAGE_SUM in half allele units, so `.5` endings too), score columns to the printed
digits.  The refusals keep the reference's wording and exit codes.  The host driver is replayed on the CPU through the
stand-in libraries (tests/harness/mock_score_sex.cc ahead of tests/harness/mock_pl2gpu.cc, injected with LD_PRELOAD as
in test_score_cols.py), and its reports must match every golden."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from oracle import plink_oracle as orc
from test_score_cols import score_file_entries_cols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
SCORE = "x_score_sex.txt.gz"
FULL = ["cols=+scoresums,+denom,+dosagesum"]
COLS = ["--score-col-nums", "3-5"]

# golden -> (command line after --bfile x, coefficient tokens (0-based), --remove-nosex, --xchr-model, no-mean-imputation, center)
CASES = {
    "x_ssx_nmi.sscore": (["--score", SCORE, "header-read", "no-mean-imputation"] + FULL + COLS, [2, 3, 4], False, 2, True, False),
    "x_ssx_nmi1.sscore": (["--score", SCORE, "header-read", "no-mean-imputation"] + FULL + COLS + ["--xchr-model", "1"], [2, 3, 4], False, 1, True, False),
    "x_ssx_rn.sscore": (["--remove-nosex", "--score", SCORE, "header-read"] + FULL + COLS, [2, 3, 4], True, 2, False, False),
    "x_ssx_rn1.sscore": (["--remove-nosex", "--score", SCORE, "header-read"] + FULL + COLS + ["--xchr-model", "1"], [2, 3, 4], True, 1, False, False),
    "x_ssx_ctr1.sscore": (["--remove-nosex", "--score", SCORE, "header-read", "center", "cols=+scoresums"] + COLS + ["--xchr-model", "1"], [2, 3, 4], True, 1, False, True),
    "x_ssx_one.sscore": (["--score", SCORE, "1", "2", "4", "header-read", "no-mean-imputation", "cols=+denom,+dosagesum", "--xchr-model", "1"], [3], False, 1, True, False),
}
VCASES = {
    "x_vsx.vscore": (["--remove-nosex", "--variant-score", "x_vscore_sex.txt", "cols=+altfreq"], 2),
    "x_vsx1.vscore": (["--remove-nosex", "--variant-score", "x_vscore_sex.txt", "cols=+altfreq", "--xchr-model", "1"], 1),
}


# ------------------------------------------------------------------------------- numpy restatement
def set_x(remove_nosex):
    """Genotypes [variant, sample], chromosome classes ('dip' / 'x' / 'y' / 'hap'), sexes, founder flags, IDs and
    alleles of set X, without its unknown-sex samples under --remove-nosex."""
    fam = [ln.split() for ln in open(os.path.join(GD, "x.fam"))]
    bim = [ln.split() for ln in open(os.path.join(GD, "x.bim"))]
    geno = orc.read_bed(os.path.join(GD, "x.bed"), len(fam))
    sex = np.array([int(t[4]) for t in fam])
    founder = np.array([t[2] == "0" and t[3] == "0" for t in fam])
    keep = sex != 0 if remove_nosex else np.ones(len(fam), dtype=bool)
    cls = np.array([orc._chr_class(b[0]) for b in bim])
    return geno[:, keep], cls, sex[keep], founder[keep], [b[1] for b in bim], [b[5] for b in bim], [b[4] for b in bim]


def class_ref_freqs(geno, cls, sex, founder):
    """Founder REF frequencies with the reference's per-class counting (chrX males once, chrY nonfemales, MT haploid)."""
    return orc.ld_ref_freqs_by_class(geno[:, founder], cls, sex[founder])


def score_report_sex(geno, cls, sex, entries, ref_freq, xchr_model=2, no_mean_imputation=False, center=False, variance_standardize=False):
    """ScoreReport on hard calls with sex-dependent ploidy (2.0/plink2_matrix_calc.cc:6682-6845, :7792-8037, report
    :8581).  A sample's named-allele dosage is the copy count on a diploid call and half of it on a haploid one (MT;
    chrY males; chrX males under --xchr-model 1); a nonmissing call adds dosage x slope + intercept, with the intercept
    -p f slope from the VARIANT's ploidy p (1 on chrY / MT, 2 elsewhere, chrX included); a missing call adds (sample
    ploidy) x f x slope and no intercept.  On chrY females add nothing and the reference also zeroes the dosage of
    unknown-sex samples (their nonmissing calls add the intercept alone); missing calls of nonfemales count as haploid.
    Missing calls, ALLELE_CT and DENOM count once per variant.  Returns ALLELE_CT, DENOM, the dosage sum in half allele
    units, and the score sums and averages as [sample, column]."""
    n = geno.shape[1]
    male, female, unknown = sex == 1, sex == 2, sex == 0
    ssum = np.zeros((n, len(entries[0][2])))
    hdos = np.zeros(n, dtype=np.int64)
    for v, aidx, coefs in entries:
        g = geno[v]
        miss = g == 3
        named = np.where(miss, 0, g if aidx == 1 else 2 - g).astype(np.int64)
        f = (1.0 - ref_freq[v]) if aidx == 1 else ref_freq[v]
        c = cls[v]
        p = 1.0 if c in ("y", "hap") else 2.0
        slope = 1.0
        if variance_standardize:
            var = (p * 0.5) * (2.0 * f * (1.0 - f))
            slope = 1.0 / np.sqrt(var) if var > orc.SMALL_EPSILON else 0.0
        icpt = (-p * f) * slope if (center or variance_standardize) else 0.0
        if c == "hap":
            hap = np.ones(n, dtype=bool)
        elif c == "y":
            hap = male
        elif c == "x" and xchr_model == 1:
            hap = male
        else:
            hap = np.zeros(n, dtype=bool)
        dose = np.where(hap, 0.5 * named, named.astype(np.float64))
        val = dose * slope + icpt
        miss_val = 0.0 if no_mean_imputation else np.where(hap | (c == "y"), 1.0, 2.0) * f * slope
        val = np.where(miss, miss_val, val)
        counted = np.where(hap, named, 2 * named)
        if c == "y":
            val = np.where(female, 0.0, np.where(unknown & ~miss, icpt, val))
            counted = np.where(male, counted, 0)
        ssum += val[:, None] * coefs[None, :]
        hdos += counted
    miss_dip, miss_hap = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
    base, y_incr, x_decr = 0, 0, 0
    for v in sorted({e[0] for e in entries}):
        c, miss = cls[v], geno[v] == 3
        if c == "hap":
            base += 1
            miss_hap += miss
        elif c == "y":
            y_incr += 1
            miss_hap += miss & ~female
        elif c == "x" and xchr_model == 1:
            base += 2
            x_decr += 1
            miss_hap += miss & male
            miss_dip += miss & ~male
        else:
            base += 2
            miss_dip += miss
    denom_full = base + np.where(female, 0, y_incr) - np.where(male, x_decr, 0)
    nallele = denom_full - 2 * miss_dip - miss_hap
    denom = nallele if no_mean_imputation else denom_full
    return nallele, denom, hdos, ssum, ssum * (1.0 / denom)[:, None]


def variant_scores_sex(geno, cls, sex, weights, ref_freq, xchr_model=2):
    """VscoreThread (2.0/plink2_matrix_calc.cc:8831-8868, :9158-9200): ALT dosage x slope (0.5 on chrY and MT, else 1),
    a missing call valued slope x 2 x ALT frequency; chrY values of nonmales zeroed, chrX male values halved under
    --xchr-model 1."""
    d = np.where(geno == 3, (2.0 * (1.0 - ref_freq))[:, None], geno.astype(np.float64))
    slope = np.where((cls == "y") | (cls == "hap"), 0.5, 1.0)
    d = d * slope[:, None]
    male = sex == 1
    d[cls == "y"] *= male[None, :]
    if xchr_model == 1:
        d[cls == "x"] *= np.where(male, 0.5, 1.0)[None, :]
    return d @ weights


def _text(path):
    return (gzip.open(path, "rt") if path.endswith(".gz") else open(path)).read()


def _table(path):
    rows = [ln.split("\t") for ln in _text(path).rstrip("\n").split("\n")]
    return rows[0], np.array(rows[1:])


def _restated(gold):
    args, cols, remove_nosex, model, no_mean, center = CASES[gold]
    geno, cls, sex, founder, ids, ref, alt = set_x(remove_nosex)
    entries, _, _ = score_file_entries_cols(os.path.join(GD, SCORE), ids, ref, alt, cols)
    return score_report_sex(geno, cls, sex, entries, class_ref_freqs(geno, cls, sex, founder), xchr_model=model, no_mean_imputation=no_mean, center=center)


@pytest.mark.parametrize("gold", sorted(CASES))
def test_restatement_matches_reference_reports(gold):
    nallele, denom, hdos, ssum, avg = _restated(gold)
    h, r = _table(os.path.join(GD, gold + ".gz"))
    names = [x[:-4] for x in h if x.endswith("_AVG")]
    assert np.array_equal(r[:, h.index("ALLELE_CT")].astype(int), nallele)
    if "DENOM" in h:
        assert np.array_equal(r[:, h.index("DENOM")].astype(int), denom)
    if "NAMED_ALLELE_DOSAGE_SUM" in h:
        assert np.array_equal((2 * r[:, h.index("NAMED_ALLELE_DOSAGE_SUM")].astype(float)).astype(int), hdos)
    for j, nm in enumerate(names):
        assert np.allclose(r[:, h.index(nm + "_AVG")].astype(float), avg[:, j], rtol=1e-5, atol=1e-9)
        if nm + "_SUM" in h:
            assert np.allclose(r[:, h.index(nm + "_SUM")].astype(float), ssum[:, j], rtol=1e-5, atol=1e-9)


def test_goldens_cover_half_dosages_and_every_sex():
    """The fixture exercises what the rules distinguish: `.5` dosage sums, and males, females and unknown sex."""
    h, r = _table(os.path.join(GD, "x_ssx_nmi1.sscore.gz"))
    assert any(x.endswith(".5") for x in r[:, h.index("NAMED_ALLELE_DOSAGE_SUM")])
    _, _, sex, _, _, _, _ = set_x(False)
    assert set(sex.tolist()) == {0, 1, 2}


def _vweights(sex_kept_iids):
    rows = [ln.split("\t") for ln in open(os.path.join(GD, "x_vscore_sex.txt")).read().rstrip("\n").split("\n")[1:]]
    by_iid = {t[1]: [float(x) for x in t[2:]] for t in rows}
    return np.array([by_iid[i] for i in sex_kept_iids])


@pytest.mark.parametrize("gold", sorted(VCASES))
def test_variant_score_restatement_matches_reference_reports(gold):
    _, model = VCASES[gold]
    geno, cls, sex, founder, _, _, _ = set_x(True)
    iids = [ln.split()[1] for ln in open(os.path.join(GD, "x.fam")) if ln.split()[4] != "0"]
    rf = class_ref_freqs(geno, cls, sex, founder)
    want = variant_scores_sex(geno, cls, sex, _vweights(iids), rf, xchr_model=model)
    h, r = _table(os.path.join(GD, gold + ".gz"))
    assert np.allclose(r[:, h.index("ALT_FREQ")].astype(float), 1.0 - rf, rtol=1e-5, atol=1e-9)
    for j, nm in enumerate(("V1", "V2")):
        assert np.allclose(r[:, h.index(nm)].astype(float), want[:, j], rtol=1e-5, atol=1e-9)


# ------------------------------------------------------------------------------- the host program
@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    """The sex-dependent score stand-in first, so its score_* symbols are the ones the host program binds."""
    d = tmp_path_factory.mktemp("mock")
    sos = []
    for name in ("mock_score_sex", "mock_pl2gpu"):
        so = str(d / (name + ".so"))
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", name + ".cc")], check=True)
        sos.append(so)
    return " ".join(sos)


def _replay(mock_so, args, out):
    env = dict(os.environ, LD_PRELOAD=mock_so, PL2_MOCK_DEVICES="1")
    return subprocess.run([BIN, "--bfile", "x"] + args + ["--out", out], capture_output=True, text=True, env=env, cwd=GD)


def _one_entry_file(tmp_path, chrom):
    """A score file naming the first variant of a chromosome by its ALT allele."""
    b = next(ln.split() for ln in open(os.path.join(GD, "x.bim")) if ln.split()[0] == chrom)
    path = tmp_path / ("one_%s.txt" % chrom)
    path.write_text("%s\t%s\t0.5\n" % (b[1], b[4]))
    return str(path)


DOMREC = "--score[-list] 'dominant' and 'recessive' modifiers cannot be used with\nhaploid chromosomes."
VARSTD = "--score[-list] 'variance-standardize' cannot be used with chrX or MT."
YNOSEX = "When both chrY variants and unknown-sex samples are present,\n--score[-list] can only be run with the 'no-mean-imputation' modifier."


@pytest.mark.parametrize("chrom,flags,msg", [
    ("X", ["dominant"], DOMREC), ("Y", ["recessive", "no-mean-imputation"], DOMREC), ("MT", ["dominant"], DOMREC),
    ("X", ["variance-standardize"], VARSTD), ("MT", ["variance-standardize"], VARSTD),
    ("Y", [], YNOSEX), ("Y", ["center"], YNOSEX),
])
def test_score_refusals_keep_the_reference_wording(mock_so, tmp_path, chrom, flags, msg):
    for model in ("1", "2"):
        r = _replay(mock_so, ["--score", _one_entry_file(tmp_path, chrom)] + flags + ["--xchr-model", model], str(tmp_path / "o"))
        assert r.returncode == 7, r.stdout + r.stderr
        assert "Error: " + msg in r.stdout


def test_allowed_forms_are_not_refused(mock_so, tmp_path):
    """chrY with variance-standardize once unknown-sex samples are gone; chrY with unknown sex and no-mean-imputation."""
    assert _replay(mock_so, ["--remove-nosex", "--score", _one_entry_file(tmp_path, "Y"), "variance-standardize"], str(tmp_path / "a")).returncode == 0
    assert _replay(mock_so, ["--score", _one_entry_file(tmp_path, "Y"), "no-mean-imputation"], str(tmp_path / "b")).returncode == 0


def test_variant_score_refuses_chr_y_with_unknown_sex(mock_so, tmp_path):
    r = _replay(mock_so, ["--variant-score", "x_vscore_sex.txt"], str(tmp_path / "o"))
    assert r.returncode == 7, r.stdout + r.stderr
    assert "Error: When chrY is present, --variant-score cannot be used with unknown-sex\nsamples." in r.stdout
    assert _replay(mock_so, ["--variant-score", "x_vscore_sex.txt", "--not-chr", "Y"], str(tmp_path / "p")).returncode == 0


@pytest.mark.parametrize("args,msg,code", [
    (["--score", SCORE, "header-read", "--xchr-model", "0"], "--xchr-model 0 (skip chrX) is not supported by plink2_b200; use --not-chr X to leave chrX out.", 63),
    (["--variant-score", "x_vscore_sex.txt", "--xchr-model", "0"], "--xchr-model 0 (skip chrX) is not supported by plink2_b200; use --not-chr X to leave chrX out.", 63),
    (["--score", SCORE, "header-read", "--xchr-model", "3"], "Invalid --xchr-model argument '3'.", 8),
    (["--score", SCORE, "header-read", "--xchr-model", "12"], "Invalid --xchr-model argument '12'.", 8),
    (["--freq", "--xchr-model", "1"], "--xchr-model must be used with --glm, --score[-list], or\n--variant-score.", 8),
])
def test_xchr_model_command_line(args, msg, code, tmp_path):
    """Refused before any device work, so no stand-in is needed."""
    r = subprocess.run([BIN, "--bfile", "x"] + args + ["--out", str(tmp_path / "o")], capture_output=True, text=True, cwd=GD)
    assert r.returncode == code, r.stdout + r.stderr
    assert "Error: " + msg in r.stdout


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
    r = _replay(mock_so, CASES[gold][0], out)
    assert r.returncode == 0, r.stdout + r.stderr
    _text_close(out + ".sscore", gold)


@pytest.mark.parametrize("gold", sorted(VCASES))
def test_variant_score_driver_replayed_on_the_cpu(mock_so, tmp_path, gold):
    out = str(tmp_path / "o")
    r = _replay(mock_so, VCASES[gold][0], out)
    assert r.returncode == 0, r.stdout + r.stderr
    _text_close(out + ".vscore", gold)
