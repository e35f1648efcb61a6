"""CPU: `--score-list`, every score file of a list scored in one report, and the 'ignore-dup-ids' modifier.

A numpy restatement of the reference's rules (each file its own score columns, named SCORE<k> by position over all the
files or by each file's header, with that file's own denominators: 2.0/plink2_matrix_calc.cc:7324, :7620-7672, :8389,
:8595-8612; 'ignore-dup-ids' :7724) is pinned to its reports on sets A and X (tests/golden/make_score_list_set.py).  The
command-line and list-file refusals keep the reference's wording and exit codes.  The host driver is replayed on the CPU
through the stand-in libraries (tests/harness/mock_score_list.cc ahead of tests/harness/mock_pl2gpu.cc, injected with
LD_PRELOAD), and its reports must match every golden, also when a small --gpu-memory splits the classes into several
passes over the genotypes."""
import glob
import os
import subprocess

import numpy as np
import pytest

from oracle import plink_oracle as orc
from test_q_score_range import load_pvals, load_ranges, zstd_decompress
from test_score_cols import score_report_cols
from test_score_sex import _table, _text_close, class_ref_freqs, score_report_sex, set_x

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")
A_LIST = ["--bfile", "a", "--score-list", "a_sl.list"]
X_LIST = ["--score-list", "x_sl.list", "header-read", "cols=+scoresums"]
X_COLS = ["--score-col-nums", "3-5"]
D_SET = ["--bed", "a.bed", "--bim", "d.bim", "--fam", "a.fam"]
QSR = ["--q-score-range", "a_qsr_mixed.ranges", "a_qsr.pvals", "header"]


def _c(args, sset, cols=(2,), mode="", no_mean=False, model=2, remove_nosex=False, qsr=False, rf=False):
    return dict(args=args, set=sset, cols=list(cols), mode=mode, no_mean=no_mean, model=model, remove_nosex=remove_nosex, qsr=qsr, rf=rf)


# run -> command line (run from tests/golden) and the restatement's settings (cols: 0-based coefficient tokens)
CASES = {
    "a_sl_plain": _c(A_LIST + ["header"], "a"),
    "a_sl_hr": _c(A_LIST + ["header-read", "cols=+scoresums"], "a"),
    "a_sl_cols": _c(A_LIST + ["header-read", "--score-col-nums", "3-7"], "a", cols=range(2, 7)),
    "a_sl_center": _c(A_LIST + ["header-read", "center"], "a", mode="center"),
    "a_sl_vs": _c(A_LIST + ["header-read", "variance-standardize", "cols=+scoresums"], "a", mode="variance-standardize"),
    "a_sl_dom": _c(A_LIST + ["header-read", "dominant"], "a", mode="dominant"),
    "a_sl_rec": _c(A_LIST + ["header-read", "recessive"], "a", mode="recessive"),
    "a_sl_nmi": _c(A_LIST + ["header-read", "no-mean-imputation", "cols=+scoresums", "--score-col-nums", "3,5"], "a", cols=(2, 4), no_mean=True),
    "a_sl_zs": _c(A_LIST + ["header", "zs"], "a"),
    "a_sl_rf": _c(A_LIST + ["header-read", "--read-freq", "a_rf.afreq"], "a", rf=True),
    "a_sl_qsr": _c(A_LIST + ["header-read", "cols=+scoresums"] + QSR, "a", qsr=True),
    "a_sl_one": _c(["--bfile", "a", "--score-list", "a_sl_one.list", "header-read"], "a"),
    "x_sl_rn1": _c(["--bfile", "x", "--remove-nosex"] + X_LIST + X_COLS + ["--xchr-model", "1"], "x", cols=(2, 3, 4), model=1, remove_nosex=True),
    "x_sl_rn2": _c(["--bfile", "x", "--remove-nosex"] + X_LIST + X_COLS + ["--xchr-model", "2"], "x", cols=(2, 3, 4), model=2, remove_nosex=True),
    "x_sl_nmi1": _c(["--bfile", "x"] + X_LIST + ["no-mean-imputation"] + X_COLS + ["--xchr-model", "1"], "x", cols=(2, 3, 4), no_mean=True, model=1),
    "d_dup_score": _c(D_SET + ["--score", "d_sl_1.txt", "header", "ignore-dup-ids"], "d"),
    "d_dup_list": _c(D_SET + ["--score-list", "d_sl.list", "header", "ignore-dup-ids", "cols=+scoresums"], "d"),
}


# ------------------------------------------------------------------------------- numpy restatement
def list_files(args):
    """The score files of a run: the first token of each list line up to the first line without one."""
    if "--score" in args:
        return [args[args.index("--score") + 1]]
    out = []
    for ln in open(os.path.join(GD, args[args.index("--score-list") + 1])):
        t = ln.split()
        if not t:
            break
        out.append(t[0])
    return out


def file_entries(path, ids, ref, alt, cols):
    """(variant index, named-allele index 0 = REF / 1 = ALT, coefficients) of a score file with a header line; IDs
    that occur more than once in the dataset are skipped ('ignore-dup-ids')."""
    idx, dup = {}, set()
    for k, v in enumerate(ids):
        if v in idx:
            dup.add(v)
        idx.setdefault(v, k)
    out = []
    for ln in open(os.path.join(GD, path)).read().split("\n")[1:]:
        t = ln.split()
        if not t or t[0] not in idx or t[0] in dup or t[1] not in (ref[idx[t[0]]], alt[idx[t[0]]]):
            continue
        k = idx[t[0]]
        out.append((k, 0 if t[1] == ref[k] else 1, np.array([float(t[c]) for c in cols])))
    return out


def score_names(run):
    """Each file's columns: SCORE<k> by position over all the files, or the file's header tokens with 'header-read'."""
    case = CASES[run]
    files = list_files(case["args"])
    if "header-read" not in case["args"]:
        return [["SCORE%d" % (f * len(case["cols"]) + j + 1) for j in range(len(case["cols"]))] for f in range(len(files))]
    return [[open(os.path.join(GD, p)).readline().split()[c] for c in case["cols"]] for p in files]


def restated(run):
    """{report suffix ('' or '.<range>'): (averages, sums)} with one [sample, column] block per file, in list order."""
    case = CASES[run]
    if case["set"] == "x":
        geno, cls, sex, founder, ids, ref, alt = set_x(case["remove_nosex"])
        rf = class_ref_freqs(geno, cls, sex, founder)
    else:
        geno = orc.read_bed(os.path.join(GD, "a.bed"), 100)
        bim = [ln.split() for ln in open(os.path.join(GD, "d.bim" if case["set"] == "d" else "a.bim"))]
        ids, ref, alt = [b[1] for b in bim], [b[5] for b in bim], [b[4] for b in bim]
        rf = orc.ref_allele_freqs(geno)
        if case["rf"]:
            ov = orc.read_freq_overrides(os.path.join(GD, "a_rf.afreq"), ids, ref, alt)
            rf = np.where(np.isfinite(ov), ov, rf)
    n, ncol = geno.shape[1], len(case["cols"])

    def report(entries):
        if not entries:
            with np.errstate(invalid="ignore", divide="ignore"):
                return np.zeros((n, ncol)) * (1.0 / np.zeros(n))[:, None], np.zeros((n, ncol))
        if case["set"] == "x":
            _, _, _, ssum, avg = score_report_sex(geno, cls, sex, entries, rf, xchr_model=case["model"], no_mean_imputation=case["no_mean"])
        else:
            _, _, _, ssum, avg = score_report_cols(geno, entries, rf, no_mean_imputation=case["no_mean"], mode=case["mode"])
        return avg, ssum

    per_file = [file_entries(p, ids, ref, alt, case["cols"]) for p in list_files(case["args"])]
    subsets = {"": per_file}
    if case["qsr"]:
        pv = load_pvals(ids, "a_qsr.pvals", 0, 1, True, False)
        subsets = {"." + nm: [[e for e in es if e[0] in pv and lb <= pv[e[0]] <= ub] for es in per_file] for nm, lb, ub in load_ranges("a_qsr_mixed.ranges")}
    out = {}
    for suffix, files in subsets.items():
        reps = [report(es) for es in files]
        out[suffix] = (np.hstack([r[0] for r in reps]), np.hstack([r[1] for r in reps]))
    return out


GOLDENS = sorted((run, suffix) for run in CASES for suffix in (["." + nm for nm, _, _ in load_ranges("a_qsr_mixed.ranges")] if CASES[run]["qsr"] else [""]))


@pytest.mark.parametrize("run,suffix", GOLDENS)
def test_restatement_matches_reference_reports(run, suffix):
    """Every file's _AVG (then _SUM) columns in list order, to the 6 printed digits; 0 / 0 averages as nan."""
    avg, ssum = restated(run)[suffix]
    h, r = _table(os.path.join(GD, "%s%s.sscore.gz" % (run, suffix)))
    names = [nm for f in score_names(run) for nm in f]
    avg_cols = [k for k, x in enumerate(h) if x.endswith("_AVG")]
    sum_cols = [k for k, x in enumerate(h) if x.endswith("_SUM") and x != "NAMED_ALLELE_DOSAGE_SUM"]
    assert [h[k] for k in avg_cols] == [nm + "_AVG" for nm in names]
    assert not {"ALLELE_CT", "DENOM", "NAMED_ALLELE_DOSAGE_SUM"} & set(h) or "--score" in CASES[run]["args"]
    assert np.allclose(r[:, avg_cols].astype(float), avg, rtol=1e-5, atol=1e-9, equal_nan=True)
    if sum_cols:
        assert [h[k] for k in sum_cols] == [nm + "_SUM" for nm in names]
        assert np.allclose(r[:, sum_cols].astype(float), ssum, rtol=1e-5, atol=1e-9)


def test_goldens_cover_the_list_forms():
    """Overlapping and disjoint files, a variant named by different alleles in two files, IDs not in the dataset, a
    file listed twice, a one-file list, and duplicated dataset IDs."""
    bim = [ln.split() for ln in open(os.path.join(GD, "a.bim"))]
    ids, ref, alt = [b[1] for b in bim], [b[5] for b in bim], [b[4] for b in bim]
    f1, f2, f3 = (file_entries("a_sl_%d.txt" % k, ids, ref, alt, [2]) for k in (1, 2, 3))
    v1, v2, v3 = ({e[0] for e in f} for f in (f1, f2, f3))
    same = {(e[0], e[1]) for e in f1}
    assert v1 & v2 and v1 & v3 and not {e[0] for e in f3 if (e[0], e[1]) in same} & v2
    assert {(e[0], 1 - e[1]) for e in f1 + f2} & {(e[0], e[1]) for e in f3}
    assert "nosuch0" in open(os.path.join(GD, "a_sl_3.txt")).read()
    assert list_files(CASES["a_sl_plain"]["args"]) == ["a_sl_1.txt", "a_sl_2.txt", "a_sl_3.txt", "a_sl_1.txt"]
    assert len(list_files(CASES["a_sl_one"]["args"])) == 1
    d_ids = [ln.split()[1] for ln in open(os.path.join(GD, "d.bim"))]
    assert len(set(d_ids)) < len(d_ids)
    _, cls, _, _, _, _, _ = set_x(False)
    assert set(cls.tolist()) == {"dip", "x", "y", "hap"}


# ------------------------------------------------------------------------------- the host program
@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    """The shared-row score stand-in first, so its score_* symbols are the ones the host program binds."""
    d = tmp_path_factory.mktemp("mock")
    sos = []
    for name in ("mock_score_list", "mock_pl2gpu", "mock_score_sex"):
        so = str(d / (name + ".so"))
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", name + ".cc")], check=True)
        sos.append(so)
    return " ".join(sos)


def _replay(mock_so, args, out, log=None):
    """--score-list runs through the shared-row stand-in, --score runs through the plain one."""
    so = mock_so.split()
    env = dict(os.environ, LD_PRELOAD=" ".join([so[2] if "--score" in args else so[0], so[1]]), PL2_MOCK_DEVICES="1")
    if log:
        env["PL2_MOCK_SCORE_LOG"] = log
    return subprocess.run([BIN] + args + ["--out", out], capture_output=True, text=True, env=env, cwd=GD)


def check_run_outputs(run, out):
    """Every report of `run` written under the prefix `out` matches its golden (6 significant digits at rtol 2e-5,
    everything else exact), and no other report was written."""
    suffixes = [s for r, s in GOLDENS if r == run]
    zs = "zs" in CASES[run]["args"]
    written = sorted(glob.glob(out + ".sscore*") + glob.glob(out + ".*.sscore*"))
    assert written == sorted("%s%s.sscore%s" % (out, s, ".zst" if zs else "") for s in suffixes)
    for s in suffixes:
        path = "%s%s.sscore" % (out, s)
        if zs:
            with open(path, "wb") as f:
                f.write(zstd_decompress(path + ".zst"))
        _text_close(path, "%s%s.sscore" % (run, s))


@pytest.mark.parametrize("run", sorted(CASES))
def test_score_driver_replayed_on_the_cpu(mock_so, tmp_path, run):
    out = str(tmp_path / "o")
    r = _replay(mock_so, CASES[run]["args"], out)
    assert r.returncode == 0, r.stdout + r.stderr
    check_run_outputs(run, out)
    if run == "a_sl_plain":
        for k, ct in enumerate([244, 255, 66, 244]):
            assert "--score-list file %d/4: %d variants processed." % (k + 1, ct) in r.stdout
        assert "Warning: --score-list: 4 entries in a_sl_3.txt were skipped due to missing variant IDs, and 3 were skipped due to mismatching allele codes." in r.stdout
        assert "--score-list: Results written to %s.sscore ." % out in r.stdout
    if run == "a_sl_qsr":
        assert "--score-list + --q-score-range: Results written to %s.<range name>.sscore ." % out in r.stdout
    if run.startswith("d_dup"):
        flag = "--score" if run == "d_dup_score" else "--score-list"
        assert "Warning: %s: 14 entries in d_sl_1.txt were skipped since their variant IDs appear multiple times in the main dataset." % flag in r.stdout


@pytest.mark.parametrize("run", ["a_sl_hr", "a_sl_qsr", "x_sl_nmi1"])
def test_classes_split_into_passes_by_gpu_memory(mock_so, tmp_path, run):
    """A 1 MiB budget holds no accumulator set next to the staging buffers: one class per pass, same reports."""
    out, log = str(tmp_path / "o"), str(tmp_path / "log")
    r = _replay(mock_so, CASES[run]["args"] + ["--gpu-memory", "1"], out, log)
    assert r.returncode == 0, r.stdout + r.stderr
    check_run_outputs(run, out)
    begins = [ln for ln in open(log).read().split("\n") if ln.startswith("begin")]
    assert len(begins) > 1 and set(begins) == {"begin 1"}
    assert "passes over the genotypes." in r.stdout
    one = str(tmp_path / "one.log")
    assert _replay(mock_so, CASES[run]["args"], str(tmp_path / "p"), one).returncode == 0
    assert [ln for ln in open(one).read().split("\n") if ln.startswith("begin")] == ["begin %d" % len(begins)]


def test_shared_variants_are_staged_once(mock_so, tmp_path):
    """One add call stages each distinct variant of all the files once; entries read their rows."""
    log = str(tmp_path / "log")
    assert _replay(mock_so, CASES["a_sl_plain"]["args"], str(tmp_path / "o"), log).returncode == 0
    adds = [tuple(map(int, ln.split()[1:])) for ln in open(log).read().split("\n") if ln.startswith("add")]
    bim = [ln.split() for ln in open(os.path.join(GD, "a.bim"))]
    ids, ref, alt = [b[1] for b in bim], [b[5] for b in bim], [b[4] for b in bim]
    per_file = [file_entries(p, ids, ref, alt, [2]) for p in list_files(CASES["a_sl_plain"]["args"])]
    assert sum(a[0] for a in adds) == len({e[0] for es in per_file for e in es})
    assert sum(a[1] for a in adds) == sum(len(es) for es in per_file)


def test_list_ends_at_its_first_blank_line(mock_so, tmp_path):
    lst = tmp_path / "l.list"
    lst.write_text("a_sl_1.txt\n a_sl_2.txt extra\n\na_sl_3.txt\n")
    r = _replay(mock_so, ["--bfile", "a", "--score-list", str(lst), "header"], str(tmp_path / "o"))
    assert r.returncode == 0, r.stdout + r.stderr
    h, _ = _table(str(tmp_path / "o.sscore"))
    assert h[-2:] == ["SCORE1_AVG", "SCORE2_AVG"] and "--score-list file 2/2: 255 variants processed." in r.stdout


def test_one_file_list_is_score(mock_so, tmp_path):
    """A one-file list writes --score's _AVG columns (stand-in sums)."""
    r = _replay(mock_so, ["--bfile", "a", "--score-list", "a_sl_one.list", "header-read", "cols=+scoresums"], str(tmp_path / "l"))
    assert r.returncode == 0, r.stdout + r.stderr
    p = _replay(mock_so, ["--bfile", "a", "--score", "a_sl_2.txt", "header-read", "cols=+scoresums"], str(tmp_path / "s"))
    assert p.returncode == 0, p.stdout + p.stderr
    hl, rl = _table(str(tmp_path / "l.sscore"))
    hs, rs = _table(str(tmp_path / "s.sscore"))
    for nm in ("BETA_AVG", "BETA_SUM"):
        assert np.array_equal(rl[:, hl.index(nm)], rs[:, hs.index(nm)])


@pytest.mark.parametrize("args,msg", [
    (A_LIST + ["list-variants"], "'list-variants[-zs]' modifier can only be used with --score, not\n--score-list."),
    (A_LIST + ["cols=+nallele"], "--score-list cannot be used with the nallele, denom, or dosagesum\ncolumn-sets."),
    (A_LIST + ["cols=+denom"], "--score-list cannot be used with the nallele, denom, or dosagesum\ncolumn-sets."),
    (A_LIST + ["cols=scoreavgs,dosagesum"], "--score-list cannot be used with the nallele, denom, or dosagesum\ncolumn-sets."),
    (A_LIST + ["header", "header-read"], "--score[-list] 'header' and 'header-read' modifiers cannot be used\ntogether."),
    (A_LIST + ["center", "dominant"], "--score[-list] 'dominant', 'recessive', 'center', and\n'variance-standardize' modifiers are mutually exclusive."),
    (A_LIST + ["center", "variance-standardize"], "--score[-list] 'dominant', 'recessive', 'center', and\n'variance-standardize' modifiers are mutually exclusive."),
    (A_LIST + ["--score", "a_sl_1.txt"], "--score-list cannot be used with --score."),
    (["--bfile", "a", "--score", "a_sl_1.txt", "--score-list", "a_sl.list"], "--score-list cannot be used with --score."),
    (A_LIST + ["se"], "not supported"),
    (["--bfile", "a", "--score-list"], "--score-list requires a filename."),
])
def test_command_line_refusals(args, msg, tmp_path):
    """Refused with code 8 before any device work, so no stand-in is needed."""
    r = subprocess.run([BIN] + args + ["--out", str(tmp_path / "o")], capture_output=True, text=True, cwd=GD)
    assert r.returncode == 8, r.stdout + r.stderr
    assert ("Error: " + msg if msg != "not supported" else msg) in r.stdout


@pytest.mark.parametrize("files,msg,code", [
    ({"l.list": ""}, "--score-list: {d}/l.list is empty.", 6),
    ({"l.list": "\nfoo.txt\n"}, "--score-list: {d}/l.list is empty.", 6),
    ({"l.list": "{d}/nofile.txt\n"}, "Failed to open {d}/nofile.txt", 3),
    ({"l.list": "{d}/s.txt\n", "s.txt": "SNP A1 B\nnosuch A 1\n"}, "--score-list: No valid variants in {d}/s.txt.", 13),
    ({"l.list": "a_sl_1.txt\n{d}/s.txt\n", "s.txt": "SNP A1 B\n\n"}, "--score-list: No valid variants in {d}/s.txt.", 13),
    ({"l.list": "a_sl_1.txt\n{d}/s.txt\n", "s.txt": "\n \n"}, "--score-list: {d}/s.txt is empty.", 6),
    ({"l.list": "a_sl_1.txt\n{d}/s.txt\n", "s.txt": "SNP A1 B\nsnp1 B\n"}, "Line 2 of {d}/s.txt has fewer tokens than expected.", 6),
    ({"l.list": "{d}/s.txt\n", "s.txt": "SNP A1 B\nsnp1 B 1\nsnp1 B 2\n"}, "--score-list: ALT1 allele for variant 'snp1' appears multiple times in {d}/s.txt-list file.", 6),
])
def test_list_file_refusals(mock_so, tmp_path, files, msg, code):
    d = str(tmp_path)
    for name, text in files.items():
        (tmp_path / name).write_text(text.format(d=d))
    r = _replay(mock_so, ["--bfile", "a", "--score-list", str(tmp_path / "l.list"), "header"], str(tmp_path / "o"))
    assert r.returncode == code, r.stdout + r.stderr
    assert "Error: " + msg.format(d=d) in r.stdout
    assert not glob.glob(str(tmp_path / "o*.sscore"))


@pytest.mark.parametrize("flag,arg", [("--score", "d_sl_1.txt"), ("--score-list", "d_sl.list")])
def test_duplicate_ids_refused_without_ignore_dup_ids(mock_so, tmp_path, flag, arg):
    """Without 'ignore-dup-ids' the first entry whose ID occurs twice in the dataset stops the run, as before."""
    r = _replay(mock_so, D_SET + [flag, arg, "header"], str(tmp_path / "o"))
    assert r.returncode == 7, r.stdout + r.stderr
    assert "Error: %s variant ID '" % flag in r.stdout and "' appears multiple times in main dataset." in r.stdout
