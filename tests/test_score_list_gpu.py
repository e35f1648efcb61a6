"""GPU: shared-row `--score` jobs (pl2gpu_score_begin_classes / _add_entries / _get_class) and the `--score-list`
command line.

(a) the library against a numpy statement of its contract at 1, 2, 9 and 33 classes and 1, 4 and 5 columns: rows read
by up to class-count entries, batches whose entries (not rows) fill the stage so that they end between rows, classes
interleaved, with and without mixed ploidy classes; (b) a rerun is bit-identical; (c) one entry per row is bit-identical
to pl2gpu_score_add_variants_classes; (d) the command line against every report of the reference; (e) a one-file list
writes --score's _AVG columns; (f) a run split into passes by a small --gpu-memory agrees with the one-pass run."""
import os
import subprocess

import numpy as np
import pytest

from plink_ng_b200.host import SCORE_DIPLOID, pack_genotypes, score_sums_classes, score_sums_entries
from test_score_list import CASES, check_run_outputs
from test_score_sex import _table
from test_score_sex_gpu import STAGE, _problem, _sexes, _want

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
ENV = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])


def _entries(row_ct, class_ct, seed):
    """Per row 1 .. max(class_ct, 2) entries (a row may have two entries of one class), classes drawn at random."""
    rng = np.random.default_rng(seed)
    per_row = rng.integers(1, max(class_ct, 2) + 1, size=row_ct)
    rows = np.repeat(np.arange(row_ct, dtype=np.uint32), per_row)
    return rows, rng.integers(0, class_ct, size=rows.size).astype(np.uint32)


def _check(got, want, score_ct):
    sums, hdos, miss_d, miss_h = got
    want_sums, want_hdos, want_d, want_h = want
    assert np.array_equal(hdos.astype(np.int64), want_hdos)
    assert np.array_equal(miss_d.astype(np.int64), want_d) and np.array_equal(miss_h.astype(np.int64), want_h)
    for j in range(score_ct):
        assert np.allclose(sums[:, j], want_sums[:, j], rtol=1e-11, atol=1e-11 * max(np.abs(want_sums[:, j]).max(), 1.0)), j


@pytest.mark.parametrize("n,score_ct,class_ct,ploidy", [(257, 1, 1, True), (257, 4, 2, False), (1000, 5, 9, True), (300, 1, 33, True), (5000, 4, 9, False), (17, 5, 33, False), (600, 5, 2, True)])
def test_library_matches_contract(gpu_ctx, n, score_ct, class_ct, ploidy):
    """(a) and (b): every class against the contract over its own entries, each reading its row's genotypes."""
    sex = _sexes(n, "mixed", seed=n)
    row_ct = (2 * STAGE + 900) // max(class_ct // 2, 1) + 700
    erows, ecls = _entries(row_ct, class_ct, seed=class_ct * 7 + score_ct)
    geno_rows = np.random.default_rng(n).choice(4, size=(row_ct, n), p=[0.45, 0.35, 0.15, 0.05]).astype(np.uint8)
    _, pcls, named, wd, wh = _problem(n, score_ct, sex, seed=n * 10 + score_ct, m=erows.size)
    if not ploidy:
        pcls[:] = SCORE_DIPLOID
    assert erows.size > 2 * STAGE and np.bincount(erows).max() > 1
    rows = pack_genotypes(geno_rows)
    kw = dict(sample_sex=sex, ploidy_classes=pcls if ploidy else None, weights4_haploid=wh if ploidy else None)
    got = score_sums_entries(gpu_ctx, rows, n, class_ct, erows, ecls, wd, named, **kw)
    geno = geno_rows[erows]
    for k in range(class_ct):
        sel = ecls == k
        _check(got[k], _want(geno[sel], sex, pcls[sel], named[sel], wd[sel], wh[sel]), score_ct)
    again = score_sums_entries(gpu_ctx, rows, n, class_ct, erows, ecls, wd, named, **kw)
    for a, b in zip(got, again):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    # the same entries over several add calls, one of them a single row
    split = score_sums_entries(gpu_ctx, rows, n, class_ct, erows, ecls, wd, named, batches=[1000, 1, row_ct - 1001], **kw)
    for k in range(class_ct):
        sel = ecls == k
        _check(split[k], _want(geno[sel], sex, pcls[sel], named[sel], wd[sel], wh[sel]), score_ct)


@pytest.mark.parametrize("n,score_ct,class_ct", [(257, 1, 1), (5000, 5, 9), (300, 4, 33)])
def test_one_entry_per_row_is_the_classes_path(gpu_ctx, n, score_ct, class_ct):
    """(c) bit-identical sums, counts and dosages."""
    sex = _sexes(n, "mixed", seed=5)
    geno, pcls, named, wd, wh = _problem(n, score_ct, sex, seed=13, m=2 * STAGE + 500)
    ecls = np.random.default_rng(class_ct).integers(0, class_ct, size=len(pcls)).astype(np.uint32)
    rows = pack_genotypes(geno)
    kw = dict(sample_sex=sex, ploidy_classes=pcls, weights4_haploid=wh)
    got = score_sums_entries(gpu_ctx, rows, n, class_ct, np.arange(len(pcls), dtype=np.uint32), ecls, wd, named, **kw)
    want = score_sums_classes(gpu_ctx, rows, n, class_ct, ecls, wd, named, **kw)
    for a, b in zip(got, want):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


def _run(golden_dir, args, out):
    r = subprocess.run([BIN] + args + ["--out", out], capture_output=True, text=True, env=ENV, cwd=golden_dir)
    assert r.returncode == 0, r.stdout + r.stderr
    return r


@pytest.mark.parametrize("run", sorted(CASES))
def test_cli_matches_reference_reports(golden_dir, tmp_path, run):
    """(d): 6 significant digits at rtol 2e-5, 0 / 0 averages exact."""
    out = str(tmp_path / "o")
    _run(golden_dir, CASES[run]["args"], out)
    check_run_outputs(run, out)


def test_one_file_list_is_score(golden_dir, tmp_path):
    """(e) the one file's entries take the same kernels in the same order: its _AVG and _SUM columns are --score's."""
    _run(golden_dir, ["--bfile", "a", "--score-list", "a_sl_one.list", "header-read", "cols=+scoresums"], str(tmp_path / "l"))
    _run(golden_dir, ["--bfile", "a", "--score", "a_sl_2.txt", "header-read", "cols=+scoresums"], str(tmp_path / "s"))
    hl, rl = _table(str(tmp_path / "l.sscore"))
    hs, rs = _table(str(tmp_path / "s.sscore"))
    for nm in ("BETA_AVG", "BETA_SUM"):
        assert np.array_equal(rl[:, hl.index(nm)], rs[:, hs.index(nm)])


@pytest.mark.parametrize("run", ["a_sl_qsr", "x_sl_nmi1"])
def test_passes_split_by_gpu_memory_agree(golden_dir, tmp_path, run):
    """(f) one class per pass against every class in one pass."""
    r = _run(golden_dir, CASES[run]["args"] + ["--gpu-memory", "1"], str(tmp_path / "g"))
    assert "passes over the genotypes." in r.stdout
    check_run_outputs(run, str(tmp_path / "g"))
    _run(golden_dir, CASES[run]["args"], str(tmp_path / "o"))
    for path in sorted(os.listdir(tmp_path)):
        if path.startswith("o.") and path.endswith(".sscore"):
            _, a = _table(str(tmp_path / path))
            _, b = _table(str(tmp_path / ("g" + path[1:])))
            assert np.allclose(a[:, 2:].astype(float), b[:, 2:].astype(float), rtol=1e-9, atol=1e-12, equal_nan=True)
