"""CPU: `--q-score-range`, one `--score` report per p-value range.

A numpy restatement of the reference's rules (2.0/plink2_matrix_calc.cc:6960-7170 for the range and data files, the
per-range counters :7877-7991 and DENOM :8389) is pinned to its reports on sets A and X
(tests/golden/make_qsr_set.py): integer columns exact, score columns to the printed digits.  The command-line and
input-file refusals keep the reference's wording and exit codes.  The host driver is replayed on the CPU through the
stand-in libraries (tests/harness/mock_qsr.cc ahead of tests/harness/mock_pl2gpu.cc, injected with LD_PRELOAD), and its
reports must match every golden."""
import ctypes as C
import glob
import os
import subprocess

import numpy as np
import pytest

from oracle import plink_oracle as orc
from test_score_cols import score_file_entries_cols
from test_score_sex import _table, _text, _text_close, class_ref_freqs, score_report_sex

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
A_SCORE = "a_score_cols.txt.gz"
X_SCORE = "x_score_sex.txt.gz"
NESTED = ["--q-score-range", "a_qsr_nested.ranges", "a_qsr.pvals", "header"]
MIXED = ["--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "header"]
X_QSR = ["--q-score-range", "x_qsr.ranges", "x_qsr.pvals"]
X_FULL = ["header-read", "cols=+scoresums,+denom,+dosagesum", "--score-col-nums", "3-5"]
A5 = [2, 3, 4, 5, 6]


def _q(ranges, data, id_col=0, val_col=1, header=False, use_min=False):
    return dict(ranges=ranges, data=data, id_col=id_col, val_col=val_col, header=header, use_min=use_min)


# run -> (command line (run from tests/golden), set, coefficient tokens (0-based), --remove-nosex, --xchr-model,
#         no-mean-imputation, variance-standardize, range / data files)
CASES = {
    "a_qsr_nest": (["--bfile", "a", "--score", A_SCORE, "1", "2", "3", "header"] + NESTED, "a", [2], False, 2, False, False, _q("a_qsr_nested.ranges", "a_qsr.pvals", header=True)),
    "a_qsr_mix": (["--bfile", "a", "--score", A_SCORE, "header-read", "cols=+scoresums"] + MIXED, "a", [2], False, 2, False, False, _q("a_qsr_mixed.ranges", "a_qsr.pvals", header=True)),
    "a_qsr_min": (["--bfile", "a", "--score", A_SCORE, "header", "--q-score-range", "a_qsr_mixed.ranges", "a_qsr_min.pvals", "3", "1", "header", "min"], "a", [2], False, 2, False, False,
                  _q("a_qsr_mixed.ranges", "a_qsr_min.pvals", id_col=2, val_col=0, header=True, use_min=True)),
    "a_qsr_cols": (["--bfile", "a", "--score", A_SCORE, "header-read", "--score-col-nums", "3-7"] + NESTED, "a", A5, False, 2, False, False, _q("a_qsr_nested.ranges", "a_qsr.pvals", header=True)),
    "a_qsr_vs": (["--bfile", "a", "--score", A_SCORE, "header-read", "variance-standardize", "cols=+scoresums", "--score-col-nums", "3-7"] + MIXED, "a", A5, False, 2, False, True,
                 _q("a_qsr_mixed.ranges", "a_qsr.pvals", header=True)),
    "a_qsr_nmi": (["--bfile", "a", "--score", A_SCORE, "header-read", "no-mean-imputation", "cols=+denom,+dosagesum,+scoresums", "--score-col-nums", "3-7"] + MIXED, "a", A5, False, 2, True, False,
                  _q("a_qsr_mixed.ranges", "a_qsr.pvals", header=True)),
    "a_qsr_zs": (["--bfile", "a", "--score", A_SCORE, "header-read", "zs"] + NESTED, "a", [2], False, 2, False, False, _q("a_qsr_nested.ranges", "a_qsr.pvals", header=True)),
    "a_qsr_lv": (["--bfile", "a", "--score", A_SCORE, "header-read", "list-variants"] + MIXED, "a", [2], False, 2, False, False, _q("a_qsr_mixed.ranges", "a_qsr.pvals", header=True)),
    "x_qsr_rn1": (["--bfile", "x", "--remove-nosex", "--score", X_SCORE] + X_FULL + ["--xchr-model", "1"] + X_QSR, "x", [2, 3, 4], True, 1, False, False, _q("x_qsr.ranges", "x_qsr.pvals")),
    "x_qsr_rn2": (["--bfile", "x", "--remove-nosex", "--score", X_SCORE] + X_FULL + ["--xchr-model", "2"] + X_QSR, "x", [2, 3, 4], True, 2, False, False, _q("x_qsr.ranges", "x_qsr.pvals")),
    "x_qsr_nmi1": (["--bfile", "x", "--score", X_SCORE, "no-mean-imputation"] + X_FULL + ["--xchr-model", "1"] + X_QSR, "x", [2, 3, 4], False, 1, True, False, _q("x_qsr.ranges", "x_qsr.pvals")),
}


# ------------------------------------------------------------------------------- numpy restatement
def load_ranges(path):
    """Range file: name, lower and upper bound; lines without two numeric bounds are skipped; lb > ub is an error."""
    out = []
    for ln in open(os.path.join(GD, path)):
        t = ln.split()
        if len(t) < 3:
            continue
        try:
            lb, ub = float(t[1]), float(t[2])
        except ValueError:
            continue
        assert lb <= ub
        out.append((t[0], lb, ub))
    return out


def load_pvals(ids, data, id_col, val_col, header, use_min):
    """Data file: {variant index: p-value}; unknown IDs and NA p-values skipped, the smallest p-value kept with 'min'."""
    idx = {v: k for k, v in enumerate(ids)}
    lines = [ln.split() for ln in open(os.path.join(GD, data)) if ln.split()]
    out = {}
    for t in lines[1:] if header else lines:
        k = idx.get(t[id_col])
        if k is None or t[val_col] in ("NA", "nan"):
            continue
        p = float(t[val_col])
        assert use_min or k not in out
        out[k] = min(p, out.get(k, p))
    return out


def set_data(name, remove_nosex):
    fam = [ln.split() for ln in open(os.path.join(GD, name + ".fam"))]
    bim = [ln.split() for ln in open(os.path.join(GD, name + ".bim"))]
    geno = orc.read_bed(os.path.join(GD, name + ".bed"), len(fam))
    sex = np.array([int(t[4]) for t in fam])
    founder = np.array([t[2] == "0" and t[3] == "0" for t in fam])
    keep = sex != 0 if remove_nosex else np.ones(len(fam), dtype=bool)
    cls = np.array([orc._chr_class(b[0]) for b in bim])
    return geno[:, keep], cls, sex[keep], founder[keep], [b[1] for b in bim], [b[5] for b in bim], [b[4] for b in bim]


def qsr_reports(run):
    """{range name: (ALLELE_CT, DENOM, dosage sum in half units, sums, averages)}: each range is scored with the score
    file's entries whose variant's p-value lies in [lb, ub]; a range without entries has zero counts and sums and
    0 x (1 / 0) averages."""
    _, sset, cols, remove_nosex, model, no_mean, vs, q = CASES[run]
    geno, cls, sex, founder, ids, ref, alt = set_data(sset, remove_nosex)
    entries, _, _ = score_file_entries_cols(os.path.join(GD, A_SCORE if sset == "a" else X_SCORE), ids, ref, alt, cols)
    rf = class_ref_freqs(geno, cls, sex, founder)
    pv = load_pvals(ids, q["data"], q["id_col"], q["val_col"], q["header"], q["use_min"])
    out = {}
    n = geno.shape[1]
    for name, lb, ub in load_ranges(q["ranges"]):
        sub = [e for e in entries if e[0] in pv and lb <= pv[e[0]] <= ub]
        if not sub:
            z = np.zeros(n, dtype=np.int64)
            with np.errstate(invalid="ignore", divide="ignore"):
                out[name] = (z, z, z, np.zeros((n, len(cols))), np.zeros((n, len(cols))) * (1.0 / z)[:, None])
            continue
        out[name] = score_report_sex(geno, cls, sex, sub, rf, xchr_model=model, no_mean_imputation=no_mean, variance_standardize=vs)
    return out


GOLDENS = sorted((run, name) for run in CASES for name, _, _ in load_ranges(CASES[run][7]["ranges"]))


@pytest.mark.parametrize("run,rng", GOLDENS)
def test_restatement_matches_reference_reports(run, rng):
    nallele, denom, hdos, ssum, avg = qsr_reports(run)[rng]
    h, r = _table(os.path.join(GD, "%s.%s.sscore.gz" % (run, rng)))
    names = [x[:-4] for x in h if x.endswith("_AVG")]
    assert np.array_equal(r[:, h.index("ALLELE_CT")].astype(int), nallele)
    if "DENOM" in h:
        assert np.array_equal(r[:, h.index("DENOM")].astype(int), denom)
    assert np.array_equal((2 * r[:, h.index("NAMED_ALLELE_DOSAGE_SUM")].astype(float)).astype(int), hdos)
    for j, nm in enumerate(names):
        assert np.allclose(r[:, h.index(nm + "_AVG")].astype(float), avg[:, j], rtol=1e-5, atol=1e-9, equal_nan=True)
        if nm + "_SUM" in h:
            assert np.allclose(r[:, h.index(nm + "_SUM")].astype(float), ssum[:, j], rtol=1e-5, atol=1e-9)


def test_goldens_cover_the_range_forms():
    """Nested ranges of growing size, a point range that holds variants, a range that holds none, 'min' changing a
    variant's range, NA p-values, unknown IDs, and every ploidy class of set X."""
    nest = qsr_reports("a_qsr_nest")
    sizes = [int(nest["S%d" % k][0].max()) for k in range(1, 7)]
    assert sizes == sorted(sizes) and sizes[0] < sizes[-1]
    mix = qsr_reports("a_qsr_mix")
    assert mix["pt"][0].max() > 0 and mix["none"][0].max() == 0
    assert "NA" in open(os.path.join(GD, "a_qsr.pvals")).read() and "unknown" in open(os.path.join(GD, "a_qsr.pvals")).read()
    ids = [ln.split()[1] for ln in open(os.path.join(GD, "a.bim"))]
    last = load_pvals(ids, "a_qsr_min.pvals", 2, 0, True, True)
    first = {}
    for t in [ln.split() for ln in open(os.path.join(GD, "a_qsr_min.pvals"))][1:]:
        first.setdefault(t[2], float(t[0]))
    assert any(first[ids[k]] != p for k, p in last.items())
    _, cls, _, _, _, _, _ = set_data("x", False)
    assert set(cls.tolist()) == {"dip", "x", "y", "hap"}


# ------------------------------------------------------------------------------- the host program
@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    """The class-split score stand-in first, so its score_* symbols are the ones the host program binds."""
    d = tmp_path_factory.mktemp("mock")
    sos = []
    for name in ("mock_qsr", "mock_pl2gpu"):
        so = str(d / (name + ".so"))
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", name + ".cc")], check=True)
        sos.append(so)
    return " ".join(sos)


def _replay(mock_so, args, out):
    env = dict(os.environ, LD_PRELOAD=mock_so, PL2_MOCK_DEVICES="1")
    return subprocess.run([BIN] + args + ["--out", out], capture_output=True, text=True, env=env, cwd=GD)


def zstd_decompress(path):
    """All frames of a .zst file through the system libzstd."""
    z = C.CDLL("libzstd.so.1")
    z.ZSTD_findFrameCompressedSize.restype = C.c_size_t
    z.ZSTD_findFrameCompressedSize.argtypes = [C.c_void_p, C.c_size_t]
    z.ZSTD_getFrameContentSize.restype = C.c_ulonglong
    z.ZSTD_getFrameContentSize.argtypes = [C.c_void_p, C.c_size_t]
    z.ZSTD_decompress.restype = C.c_size_t
    z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    raw = open(path, "rb").read()
    buf = C.create_string_buffer(raw, len(raw))
    base = C.addressof(buf)
    out, off = b"", 0
    while off < len(raw):
        fsz = z.ZSTD_findFrameCompressedSize(base + off, len(raw) - off)
        n = z.ZSTD_getFrameContentSize(base + off, fsz)
        dst = C.create_string_buffer(max(int(n), 1))
        assert z.ZSTD_decompress(dst, n, base + off, fsz) == n
        out += dst.raw[:n]
        off += fsz
    return out


def check_run_outputs(run, out):
    """Every range's report of `run` written under the prefix `out` matches its golden (6 significant digits at rtol
    2e-5, everything else exact), and no other report was written."""
    names = [nm for nm, _, _ in load_ranges(CASES[run][7]["ranges"])]
    zs = "zs" in CASES[run][0]
    written = sorted(glob.glob(out + ".*.sscore*"))
    assert written == sorted("%s.%s.sscore%s" % (out, nm, ".zst" if zs else "") for nm in names)
    for nm in names:
        path = "%s.%s.sscore" % (out, nm)
        if zs:
            with open(path, "wb") as f:
                f.write(zstd_decompress(path + ".zst"))
        _text_close(path, "%s.%s.sscore" % (run, nm))
    if "list-variants" in CASES[run][0]:
        assert open(out + ".sscore.vars").read() == _text(os.path.join(GD, run + ".sscore.vars.gz"))


@pytest.mark.parametrize("run", sorted(CASES))
def test_score_driver_replayed_on_the_cpu(mock_so, tmp_path, run):
    out = str(tmp_path / "o")
    r = _replay(mock_so, CASES[run][0], out)
    assert r.returncode == 0, r.stdout + r.stderr
    check_run_outputs(run, out)
    if run == "a_qsr_mix":
        assert "--q-score-range: 5 ranges and 927 variants loaded." in r.stdout
        assert "Warning: 11 lines skipped in --q-score-range data file." in r.stdout
        assert "--score + --q-score-range: Results written to %s.<range name>.sscore ." % out in r.stdout


BASE = ["--bfile", "a", "--score", A_SCORE, "header-read"]


@pytest.mark.parametrize("args,msg,code", [
    (["--bfile", "a", "--freq", "--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals"], "--q-score-range cannot be used without --score[-list].", 8),
    (BASE + ["--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "1", "2", "3"], "--q-score-range takes at most two numeric arguments.", 8),
    (BASE + ["--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "2", "2"], "Identical --q-score-range column indexes.", 8),
    (BASE + ["--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "maximum"], "Invalid --q-score-range argument 'maximum'.", 8),
    (BASE + ["--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "0"], "Invalid --q-score-range argument '0'.", 8),
    (BASE + ["--q-score-range", "a_qsr_mixed.ranges"], "--q-score-range requires at least 2 arguments.", 8),
])
def test_command_line_refusals(args, msg, code, tmp_path):
    """Refused before any device work, so no stand-in is needed."""
    r = subprocess.run([BIN] + args + ["--out", str(tmp_path / "o")], capture_output=True, text=True, cwd=GD)
    assert r.returncode == code, r.stdout + r.stderr
    assert "Error: " + msg in r.stdout


def _files(tmp_path, ranges, data):
    rp, dp = tmp_path / "r.txt", tmp_path / "d.txt"
    rp.write_text(ranges)
    dp.write_text(data)
    return str(rp), str(dp)


@pytest.mark.parametrize("ranges,data,extra,msg,code", [
    ("A 0 0.5\nB 0.6 0.2\n", "snp1 0.1\n", [], "Upper bound < lower bound on line 2 of --q-score-range range file.", 6),
    ("A x 0.5\nshort\n", "snp1 0.1\n", [], "Empty --q-score-range range file.", 7),
    ("A 0 0.5\n", "snp1 0.1\nsnp2 abc\n", [], "Invalid value 'abc' on line 2 of --q-score-range data file.", 6),
    ("A 0 0.5\n", "snp1 0.1\nsnp1 0.2\n", [], "Duplicate variant ID 'snp1' in --q-score-range data file.", 6),
    ("A 0 0.5\n", "nosuch 0.1\nsnp1 NA\n", [], "No valid entries in --q-score-range data file.", 7),
    ("A 0 0.5\n", "snp1 0.1\nsnp2\n", [], "Line 2 of --q-score-range data file has fewer tokens than expected.", 7),
    ("A 0 0.5\n", "", ["header"], "Empty --q-score-range data file.", 6),
])
def test_input_file_refusals(mock_so, tmp_path, ranges, data, extra, msg, code):
    rp, dp = _files(tmp_path, ranges, data)
    r = _replay(mock_so, BASE + ["--q-score-range", rp, dp] + extra, str(tmp_path / "o"))
    assert r.returncode == code, r.stdout + r.stderr
    assert "Error: " + msg in r.stdout
    assert not glob.glob(str(tmp_path / "o.*.sscore"))


def test_min_keeps_the_smallest_p_value(mock_so, tmp_path):
    """A variant listed twice lands in the range of its smaller p-value under 'min'; unknown IDs are counted."""
    rp, dp = _files(tmp_path, "lo 0 0.2\nhi 0.5 1\n", "snp1 0.9\nsnp1 0.1\nnosuch 0.1\nsnp2 0.7\n")
    r = _replay(mock_so, BASE + ["--q-score-range", rp, dp, "min"], str(tmp_path / "o"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "--q-score-range: 2 ranges and 2 variants loaded." in r.stdout
    assert "Warning: 1 line skipped in --q-score-range data file." in r.stdout
    ids = [ln.split()[1] for ln in open(os.path.join(GD, "a.bim"))]
    entries, _, _ = score_file_entries_cols(os.path.join(GD, A_SCORE), ids, [ln.split()[5] for ln in open(os.path.join(GD, "a.bim"))], [ln.split()[4] for ln in open(os.path.join(GD, "a.bim"))], [2])
    scored = {ids[e[0]] for e in entries}
    for rng, snp in (("lo", "snp1"), ("hi", "snp2")):
        h, rows = _table(str(tmp_path / ("o.%s.sscore" % rng)))
        want = 2 if snp in scored else 0
        assert set(rows[:, h.index("ALLELE_CT")].astype(int).tolist()) <= {want, want - 2}


def test_plain_score_unchanged_by_the_class_path(mock_so, tmp_path):
    """One range holding every scored variant reports what plain --score reports, byte for byte (stand-in sums)."""
    ids = [ln.split()[1] for ln in open(os.path.join(GD, "a.bim"))]
    rp, dp = _files(tmp_path, "all 0 1\n", "".join("%s 0.5\n" % i for i in ids))
    args = BASE + ["cols=+scoresums,+denom", "--score-col-nums", "3-7"]
    r = _replay(mock_so, args + ["--q-score-range", rp, dp], str(tmp_path / "q"))
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ, LD_PRELOAD=mock_so.replace("mock_qsr.so", "mock_score_sex.so"), PL2_MOCK_DEVICES="1")
    so = mock_so.split()[0].replace("mock_qsr.so", "mock_score_sex.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", "mock_score_sex.cc")], check=True)
    p = subprocess.run([BIN] + args + ["--out", str(tmp_path / "p")], capture_output=True, text=True, env=env, cwd=GD)
    assert p.returncode == 0, p.stdout + p.stderr
    assert open(str(tmp_path / "q.all.sscore")).read() == open(str(tmp_path / "p.sscore")).read()
