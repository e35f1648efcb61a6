"""GPU: several `--score` coefficient columns in one device pass (pl2gpu_score_begin_cols).

(a) the library against the numpy restatement at column counts around the launch group width, over two staging
batches; (b) every column of a several-column job bit-identical to a one-column job of that column; (c) the command
line against the reference's reports; (d) one selected column against the three-number form; (e) the PC projection
of set A with the reference's allele weights."""
import os
import subprocess

import numpy as np
import pytest

from oracle import plink_oracle as orc
from plink_ng_b200.host import pack_genotypes, score_sums, score_sums_cols
from test_score_cols import CASES, _text, score_report_cols

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
ENV = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
G = 4  # score columns per launch (kScoreGroup in score.cu)
CODES = {("", 0): 0x06, ("", 1): 0x24, ("dominant", 0): 0x05, ("dominant", 1): 0x14, ("recessive", 0): 0x01, ("recessive", 1): 0x10}


def _problem(n, m, score_ct, seed):
    """Entries over m variants, each variant scored for one or both alleles (mixed REF / ALT naming), with additive,
    dominant and recessive dosage codes; coefficient columns include an all-zero one and all-zero rows."""
    rng = np.random.default_rng(seed)
    geno = rng.choice(4, size=(m, n), p=[0.45, 0.35, 0.17, 0.03]).astype(np.uint8)
    ref_freq = orc.ref_allele_freqs(geno)
    entries = []
    for v in range(m):
        for aidx in ((0, 1) if v % 11 == 0 else (int(rng.integers(0, 2)),)):
            entries.append((v, aidx))
    coefs = rng.normal(size=(len(entries), score_ct))
    coefs[:, score_ct // 2] = 0.0
    coefs[::13] = 0.0
    modes = rng.choice(["", "dominant", "recessive"], size=len(entries))
    w4 = np.zeros((len(entries), score_ct, 4))
    d4 = np.zeros(len(entries), dtype=np.uint8)
    for k, (v, aidx) in enumerate(entries):
        code = CODES[(modes[k], aidx)]
        dose = np.array([(code >> (2 * c)) & 3 for c in range(3)], dtype=np.float64)
        f = (1.0 - ref_freq[v]) if aidx else ref_freq[v]
        miss = (f if modes[k] else 2.0 * f)
        w4[k, :, :3] = coefs[k][:, None] * dose[None, :]
        w4[k, :, 3] = coefs[k] * miss
        d4[k] = code
    rows = pack_genotypes(geno)[[e[0] for e in entries]]
    return geno, entries, modes, coefs, ref_freq, rows, w4, d4


def _want(geno, entries, modes, coefs, ref_freq):
    """Per-mode restatement, summed over the modes (each entry in exactly one)."""
    n, sc = geno.shape[1], coefs.shape[1]
    ssum, dos = np.zeros((n, sc)), np.zeros(n, dtype=np.int64)
    for mode in ("", "dominant", "recessive"):
        sel = [k for k in range(len(entries)) if modes[k] == mode]
        if sel:
            _, _, d, s, _ = score_report_cols(geno, [(entries[k][0], entries[k][1], coefs[k]) for k in sel], ref_freq, mode=mode)
            ssum += s
            dos += d
    return ssum, dos, (geno[[e[0] for e in entries]] == 3).sum(axis=0)  # the library counts missing calls per entry


@pytest.mark.parametrize("score_ct", [1, G - 1, G, G + 1, 2 * G + 1, 64])
@pytest.mark.parametrize("n", [257, 5000])
def test_library_matches_restatement_and_one_column_jobs(gpu_ctx, n, score_ct):
    """(a) and (b): 18,000+ entries = two staging batches of several chunks each."""
    m = 16600
    geno, entries, modes, coefs, ref_freq, rows, w4, d4 = _problem(n, m, score_ct, seed=n + score_ct)
    assert len(entries) > 16384
    sums, dos, miss = score_sums_cols(gpu_ctx, rows, n, w4, d4)
    want_sum, want_dos, want_miss = _want(geno, entries, modes, coefs, ref_freq)
    assert np.array_equal(dos.astype(np.int64), want_dos) and np.array_equal(miss.astype(np.int64), want_miss)
    for j in range(score_ct):
        assert np.allclose(sums[:, j], want_sum[:, j], rtol=1e-11, atol=1e-11 * max(np.abs(want_sum[:, j]).max(), 1.0))
    for j in sorted({0, score_ct // 2, score_ct - 1, min(G, score_ct - 1)}):
        one, one_dos, one_miss = score_sums(gpu_ctx, rows, n, w4[:, j, :], d4)
        assert np.array_equal(sums[:, j], one), j  # same adds in the same order as a one-column job
        assert np.array_equal(dos, one_dos) and np.array_equal(miss, one_miss)
    again, _, _ = score_sums_cols(gpu_ctx, rows, n, w4, d4)
    assert np.array_equal(sums, again)


def test_every_column_is_bit_identical_to_its_one_column_job(gpu_ctx):
    """(b) for every column of a job that spans several launch groups and a partial last group."""
    n, m, score_ct = 1000, 17000, 2 * G + 3
    _, _, _, _, _, rows, w4, d4 = _problem(n, m, score_ct, seed=7)
    sums, dos, miss = score_sums_cols(gpu_ctx, rows, n, w4, d4)
    for j in range(score_ct):
        one, one_dos, one_miss = score_sums(gpu_ctx, rows, n, np.ascontiguousarray(w4[:, j, :]), d4)
        assert np.array_equal(sums[:, j], one), j
        assert np.array_equal(dos, one_dos) and np.array_equal(miss, one_miss)


def _table(path):
    rows = [ln.split("\t") for ln in _text(path).rstrip("\n").split("\n")]
    return rows[0], rows[1:]


def _run(golden_dir, args, out):
    r = subprocess.run([BIN, "--bfile", os.path.join(golden_dir, "a")] + args + ["--out", out], capture_output=True, text=True, env=ENV, cwd=golden_dir)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


@pytest.mark.parametrize("gold", sorted(CASES))
def test_cli_matches_reference_report(golden_dir, tmp_path, gold):
    """(c) and (e): integer columns exact, float columns to the printed digits and >= 97 % text-identical."""
    out = str(tmp_path / "s")
    _run(golden_dir, CASES[gold][6], out)
    got_h, got = _table(out + ".sscore")
    ref_h, ref = _table(os.path.join(golden_dir, gold + ".gz"))
    assert got_h == ref_h and len(got) == len(ref)
    is_float = [h.endswith("_AVG") or h.endswith("_SUM") for h in ref_h]
    same_text = 0
    for g, w in zip(got, ref):
        for col, fl in enumerate(is_float):
            if not fl:
                assert g[col] == w[col]
            else:
                assert np.isclose(float(g[col]), float(w[col]), rtol=2e-5, atol=2e-9)
                same_text += g[col] == w[col]
    assert same_text >= 0.97 * len(ref) * sum(is_float)


def test_five_header_named_columns_in_one_report(golden_dir, tmp_path):
    out = str(tmp_path / "s")
    _run(golden_dir, ["--score", "a_score_cols.txt.gz", "header-read", "--score-col-nums", "3-7"], out)
    h, _ = _table(out + ".sscore")
    assert h[-5:] == ["BETA_AVG", "NEG_AVG", "ZERO_AVG", "MIX_AVG", "HALF_AVG"]


@pytest.mark.parametrize("k", [3, 4, 6])
def test_one_selected_column_is_the_three_number_form(golden_dir, tmp_path, k):
    """(d)"""
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    _run(golden_dir, ["--score", "a_score_cols.txt.gz", "header-read", "cols=+scoresums", "--score-col-nums", str(k)], a)
    _run(golden_dir, ["--score", "a_score_cols.txt.gz", "1", "2", str(k), "header-read", "cols=+scoresums"], b)
    assert open(a + ".sscore", "rb").read() == open(b + ".sscore", "rb").read()


def test_variant_score_column_selection(golden_dir, tmp_path):
    out = str(tmp_path / "v")
    _run(golden_dir, ["--variant-score", "a_vscore_weights.txt", "--vscore-col-nums", "3"], out)
    got_h, got = _table(out + ".vscore")
    ref_h, ref = _table(os.path.join(golden_dir, "a_vsc.vscore.gz"))
    assert got_h == ref_h and len(got) == len(ref)
    for g, w in zip(got, ref):
        assert g[:-1] == w[:-1] and np.isclose(float(g[-1]), float(w[-1]), rtol=2e-5, atol=1e-9)
