"""GPU: `--score` entries with sex-dependent ploidy (pl2gpu_score_set_sex / _add_variants_ploidy / _get_ploidy) and
the sex-chromosome `--score` / `--variant-score` command lines.

(a) the library against a numpy statement of its contract at sample counts around the 16-sample word and the
128-word CTA, in all-male and all-female views, at 1, 4, 5 and 9 columns (around the launch group of four), with
runs of the four ploidy classes mixed across staging batches; (b) a rerun is bit-identical; (c) a job of diploid
entries only gives exactly the sums of the plain path; (d) the command line against the reference's reports."""
import os
import subprocess

import numpy as np
import pytest

from plink_ng_b200.host import SCORE_CHR_X_MALE_HAPLOID, SCORE_CHR_Y, SCORE_DIPLOID, SCORE_HAPLOID_ALL, pack_genotypes, score_sums_cols, score_sums_ploidy
from test_score_sex import CASES, VCASES, _text

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
ENV = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
STAGE = 16384  # entries per staging batch (kScoreStageVariants in score.cu)


def _problem(n, score_ct, sex, seed, m=STAGE + 1700):
    """m entries in runs of 1 .. 3000 entries of one ploidy class, the four classes in turn (so every staging batch
    holds several runs and a run straddles the batch boundary); diploid runs mix additive, dominant and recessive
    entries, the others are REF- or ALT-named additive entries."""
    rng = np.random.default_rng(seed)
    geno = rng.choice(4, size=(m, n), p=[0.45, 0.35, 0.15, 0.05]).astype(np.uint8)
    classes = np.zeros(m, dtype=np.uint8)
    order = rng.permutation(4)
    k, r = 0, 0
    while k < m:
        run = int(rng.integers(1, 3000))
        classes[k:k + run] = order[r % 4]
        k += run
        r += 1
    named = np.where(rng.random(m) < 0.5, 0x24, 0x06).astype(np.uint8)
    dip = classes == SCORE_DIPLOID
    named[dip] = rng.choice(np.array([0x24, 0x06, 0x14, 0x05, 0x10, 0x01], dtype=np.uint8), size=int(dip.sum()))
    wd = rng.normal(size=(m, score_ct, 4))
    wh = rng.normal(size=(m, score_ct, 4))
    wd[::17] = 0.0
    return geno, classes, named, wd, wh


def _want(geno, sex, classes, named, wd, wh):
    """The contract of include/plink2_b200.h: per entry and sample the first or second table or nothing, dosages in
    half allele units, missing calls diploid or haploid.  fp64 sums as one-hot matrix products."""
    m, n = geno.shape
    male, female = sex == 1, sex == 2
    hap = np.zeros((m, n), dtype=bool)
    skip = np.zeros((m, n), dtype=bool)
    hap[classes == SCORE_HAPLOID_ALL] = True
    hap[classes == SCORE_CHR_Y] = male
    hap[classes == SCORE_CHR_X_MALE_HAPLOID] = male
    skip[classes == SCORE_CHR_Y] = female
    sums = np.zeros((n, wd.shape[1]))
    for e0 in range(0, m, 2048):  # entry blocks keep the one-hot operands small
        sl = slice(e0, e0 + 2048)
        for code in range(4):
            at = geno[sl] == code
            sums += (at & ~hap[sl] & ~skip[sl]).T.astype(np.float64) @ wd[sl, :, code] + (at & hap[sl]).T.astype(np.float64) @ wh[sl, :, code]
    dose = (named[:, None] >> (2 * np.minimum(geno, 2))) & 3
    dose = np.where(geno == 3, 0, dose).astype(np.int64)
    ychr = (classes == SCORE_CHR_Y)[:, None]
    counted = np.where(hap, dose, np.where(ychr, 0, 2 * dose)) * ~skip
    miss = geno == 3
    miss_hap = (miss & (hap | (ychr & ~skip))).sum(axis=0)
    miss_dip = (miss & ~hap & ~ychr).sum(axis=0)
    return sums, counted.sum(axis=0), miss_dip, miss_hap


def _sexes(n, view, seed):
    if view == "male":
        return np.ones(n, dtype=np.uint8)
    if view == "female":
        return np.full(n, 2, dtype=np.uint8)
    return np.random.default_rng(seed).choice(3, size=n, p=[0.1, 0.45, 0.45]).astype(np.uint8)


@pytest.mark.parametrize("n,score_ct,view", [(1, 1, "mixed"), (15, 4, "mixed"), (16, 5, "mixed"), (17, 9, "mixed"), (33, 1, "mixed"), (257, 4, "mixed"), (5000, 5, "mixed"),
                                             (257, 5, "male"), (257, 9, "female"), (1, 4, "male")])
def test_library_matches_contract(gpu_ctx, n, score_ct, view):
    """(a) and (b)"""
    sex = _sexes(n, view, seed=n)
    geno, classes, named, wd, wh = _problem(n, score_ct, sex, seed=n * 10 + score_ct)
    assert len(classes) > STAGE and set(classes[:STAGE].tolist()) == {0, 1, 2, 3}
    rows = pack_genotypes(geno)
    sums, hdos, miss_d, miss_h = score_sums_ploidy(gpu_ctx, rows, n, sex, classes, wd, wh, named)
    want_sums, want_hdos, want_d, want_h = _want(geno, sex, classes, named, wd, wh)
    assert np.array_equal(hdos.astype(np.int64), want_hdos)
    assert np.array_equal(miss_d.astype(np.int64), want_d) and np.array_equal(miss_h.astype(np.int64), want_h)
    for j in range(score_ct):
        assert np.allclose(sums[:, j], want_sums[:, j], rtol=1e-11, atol=1e-11 * max(np.abs(want_sums[:, j]).max(), 1.0)), j
    again = score_sums_ploidy(gpu_ctx, rows, n, sex, classes, wd, wh, named)
    assert np.array_equal(sums, again[0]) and all(np.array_equal(a, b) for a, b in zip((hdos, miss_d, miss_h), again[1:]))


@pytest.mark.parametrize("n,score_ct", [(257, 1), (5000, 5)])
def test_diploid_only_job_is_the_plain_path(gpu_ctx, n, score_ct):
    """(c) bit-identical sums, the same missing counts and twice the dosage sums."""
    sex = _sexes(n, "mixed", seed=3)
    geno, classes, named, wd, wh = _problem(n, score_ct, sex, seed=11)
    rng = np.random.default_rng(5)
    named = rng.choice(np.array([0x24, 0x06, 0x14, 0x05, 0x10, 0x01], dtype=np.uint8), size=len(named))
    classes[:] = SCORE_DIPLOID
    rows = pack_genotypes(geno)
    sums, hdos, miss_d, miss_h = score_sums_ploidy(gpu_ctx, rows, n, sex, classes, wd, wh, named)
    plain, dos, miss = score_sums_cols(gpu_ctx, rows, n, wd, named)
    assert np.array_equal(sums, plain)
    assert np.array_equal(hdos, 2 * dos) and np.array_equal(miss_d, miss) and not miss_h.any()


def _table(path):
    rows = [ln.split("\t") for ln in _text(path).rstrip("\n").split("\n")]
    return rows[0], rows[1:]


def _run(golden_dir, args, out):
    r = subprocess.run([BIN, "--bfile", os.path.join(golden_dir, "x")] + args + ["--out", out], capture_output=True, text=True, env=ENV, cwd=golden_dir)
    assert r.returncode == 0, r.stdout + r.stderr


def _compare(got_path, gold_path, is_float):
    got_h, got = _table(got_path)
    ref_h, ref = _table(gold_path)
    assert got_h == ref_h and len(got) == len(ref)
    flt = [is_float(h) for h in ref_h]
    same_text = 0
    for g, w in zip(got, ref):
        for col, fl in enumerate(flt):
            if not fl:
                assert g[col] == w[col]  # IDs, phenotype, ALLELE_CT, DENOM, NAMED_ALLELE_DOSAGE_SUM, variant columns: exact
            else:
                assert np.isclose(float(g[col]), float(w[col]), rtol=2e-5, atol=2e-9)  # 6 significant digits printed
                same_text += g[col] == w[col]
    assert same_text >= 0.97 * len(ref) * sum(flt)  # fp64 sums in a different order: a last printed digit may move


@pytest.mark.parametrize("gold", sorted(CASES))
def test_score_cli_matches_reference_report(golden_dir, tmp_path, gold):
    """(d)"""
    out = str(tmp_path / "s")
    _run(golden_dir, CASES[gold][0], out)
    _compare(out + ".sscore", os.path.join(golden_dir, gold + ".gz"), lambda h: h.endswith("_AVG") or h.endswith("_SUM"))


@pytest.mark.parametrize("gold", sorted(VCASES))
def test_variant_score_cli_matches_reference_report(golden_dir, tmp_path, gold):
    """(d): ALT_FREQ from the per-class founder counting, exact as printed."""
    out = str(tmp_path / "v")
    _run(golden_dir, VCASES[gold][0], out)
    _compare(out + ".vscore", os.path.join(golden_dir, gold + ".gz"), lambda h: h in ("V1", "V2"))
