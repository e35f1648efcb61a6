"""GPU: class-split `--score` jobs (pl2gpu_score_begin_classes / _add_variants_classes / _get_class) and the
`--q-score-range` command line.

(a) the library against a numpy statement of its contract at 1, 2, 9 and 33 classes and 1, 4 and 5 columns, with the
classes interleaved across two staging batches, with and without mixed ploidy classes; (b) a rerun is bit-identical;
(c) a one-class job gives exactly the sums of the plain path, with and without ploidy classes; (d) the command line
against every report of the reference; (e) one range holding every entry writes plain --score's report byte for byte."""
import os
import subprocess

import numpy as np
import pytest

from plink_ng_b200.host import SCORE_DIPLOID, pack_genotypes, score_sums_classes, score_sums_cols, score_sums_ploidy
from test_q_score_range import CASES, check_run_outputs
from test_score_sex_gpu import STAGE, _problem, _sexes, _want

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
ENV = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])


def _classes(m, class_ct, seed):
    """Entry classes in short runs (1 .. 399 entries) that go through the classes in shuffled rounds, so every staging
    batch holds every class in several pieces."""
    rng = np.random.default_rng(seed)
    out = np.empty(m, dtype=np.uint32)
    order = np.concatenate([rng.permutation(class_ct) for _ in range(m // class_ct + 1)])
    k, r = 0, 0
    while k < m:
        run = int(rng.integers(1, min(400, 1 + STAGE // (2 * class_ct))))
        out[k:k + run] = order[r]
        k += run
        r += 1
    return out


def _check(got, want, score_ct):
    sums, hdos, miss_d, miss_h = got
    want_sums, want_hdos, want_d, want_h = want
    assert np.array_equal(hdos.astype(np.int64), want_hdos)
    assert np.array_equal(miss_d.astype(np.int64), want_d) and np.array_equal(miss_h.astype(np.int64), want_h)
    for j in range(score_ct):
        assert np.allclose(sums[:, j], want_sums[:, j], rtol=1e-11, atol=1e-11 * max(np.abs(want_sums[:, j]).max(), 1.0)), j


@pytest.mark.parametrize("n,score_ct,class_ct,ploidy", [(257, 1, 1, True), (257, 4, 2, False), (1000, 5, 9, True), (300, 1, 33, True), (5000, 4, 9, False), (17, 5, 33, False), (600, 5, 2, True)])
def test_library_matches_contract(gpu_ctx, n, score_ct, class_ct, ploidy):
    """(a) and (b): every class against the contract over its own entries."""
    sex = _sexes(n, "mixed", seed=n)
    geno, pcls, named, wd, wh = _problem(n, score_ct, sex, seed=n * 10 + score_ct, m=2 * STAGE + 900)
    if not ploidy:
        pcls[:] = SCORE_DIPLOID
    ecls = _classes(len(pcls), class_ct, seed=class_ct)
    assert len(set(ecls[:STAGE].tolist())) == class_ct and len(set(ecls[STAGE:2 * STAGE].tolist())) == class_ct
    rows = pack_genotypes(geno)
    got = score_sums_classes(gpu_ctx, rows, n, class_ct, ecls, wd, named, sample_sex=sex, ploidy_classes=pcls if ploidy else None, weights4_haploid=wh if ploidy else None)
    for k in range(class_ct):
        sel = ecls == k
        _check(got[k], _want(geno[sel], sex, pcls[sel], named[sel], wd[sel], wh[sel]), score_ct)
    again = score_sums_classes(gpu_ctx, rows, n, class_ct, ecls, wd, named, sample_sex=sex, ploidy_classes=pcls if ploidy else None, weights4_haploid=wh if ploidy else None)
    for a, b in zip(got, again):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_classes_split_over_several_calls(gpu_ctx):
    """Add calls of uneven sizes, one of them all one class, accumulate as one call does (to the contract)."""
    n, score_ct, class_ct = 400, 4, 5
    sex = _sexes(n, "mixed", seed=1)
    geno, pcls, named, wd, wh = _problem(n, score_ct, sex, seed=2, m=STAGE + 3000)
    ecls = _classes(len(pcls), class_ct, seed=3)
    ecls[100:2100] = 3
    got = score_sums_classes(gpu_ctx, pack_genotypes(geno), n, class_ct, ecls, wd, named, sample_sex=sex, ploidy_classes=pcls, weights4_haploid=wh, batches=[100, 2000, len(pcls) - 2100])
    for k in range(class_ct):
        sel = ecls == k
        _check(got[k], _want(geno[sel], sex, pcls[sel], named[sel], wd[sel], wh[sel]), score_ct)


@pytest.mark.parametrize("n,score_ct", [(257, 1), (5000, 5)])
def test_one_class_job_is_the_plain_path(gpu_ctx, n, score_ct):
    """(c) bit-identical to pl2gpu_score_add_variants (diploid) and to pl2gpu_score_add_variants_ploidy."""
    sex = _sexes(n, "mixed", seed=3)
    geno, pcls, named, wd, wh = _problem(n, score_ct, sex, seed=11)
    rows = pack_genotypes(geno)
    ecls = np.zeros(len(pcls), dtype=np.uint32)
    sums, hdos, miss_d, miss_h = score_sums_classes(gpu_ctx, rows, n, 1, ecls, wd, named, sample_sex=sex, ploidy_classes=pcls, weights4_haploid=wh)[0]
    p_sums, p_hdos, p_d, p_h = score_sums_ploidy(gpu_ctx, rows, n, sex, pcls, wd, wh, named)
    assert np.array_equal(sums, p_sums) and np.array_equal(hdos, p_hdos) and np.array_equal(miss_d, p_d) and np.array_equal(miss_h, p_h)
    sums, hdos, miss_d, miss_h = score_sums_classes(gpu_ctx, rows, n, 1, ecls, wd, named)[0]
    plain, dos, miss = score_sums_cols(gpu_ctx, rows, n, wd, named)
    assert np.array_equal(sums, plain) and np.array_equal(hdos, 2 * dos) and np.array_equal(miss_d, miss) and not miss_h.any()


@pytest.mark.parametrize("run", sorted(CASES))
def test_cli_matches_reference_reports(golden_dir, tmp_path, run):
    """(d): 6 significant digits at rtol 2e-5, integer columns and 0 / 0 averages exact."""
    out = str(tmp_path / "q")
    r = subprocess.run([BIN] + CASES[run][0] + ["--out", out], capture_output=True, text=True, env=ENV, cwd=golden_dir)
    assert r.returncode == 0, r.stdout + r.stderr
    check_run_outputs(run, out)


@pytest.mark.parametrize("mods", [["cols=+scoresums,+denom"], ["variance-standardize", "cols=+scoresums"], ["no-mean-imputation", "cols=+denom,+dosagesum,+scoresums"]])
def test_one_range_over_every_entry_is_plain_score(golden_dir, tmp_path, mods):
    """(e) byte-identical reports: every entry in one class takes the plain path's device work."""
    ids = [ln.split()[1] for ln in open(os.path.join(golden_dir, "a.bim"))]
    rp, dp = tmp_path / "r.txt", tmp_path / "d.txt"
    rp.write_text("all 0 1\n")
    dp.write_text("".join("%s 0.5\n" % i for i in ids))
    args = ["--bfile", "a", "--score", "a_score_cols.txt.gz", "header-read"] + mods + ["--score-col-nums", "3-7"]
    for extra, out in ((["--q-score-range", str(rp), str(dp)], "q"), ([], "p")):
        r = subprocess.run([BIN] + args + extra + ["--out", str(tmp_path / out)], capture_output=True, text=True, env=ENV, cwd=golden_dir)
        assert r.returncode == 0, r.stdout + r.stderr
    assert open(str(tmp_path / "q.all.sscore")).read() == open(str(tmp_path / "p.sscore")).read()
