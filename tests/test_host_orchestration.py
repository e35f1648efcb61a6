"""CPU: the HOST ORCHESTRATION of plink2_b200 around the device calls, replayed without a GPU.  A test-only stand-in
for the handful of libpl2gpu entry points the LD-prune driver uses (tests/harness/mock_pl2gpu.cc: plain-loop pair
decisions and genotype counts; the greedy walk is the product's own exported pl2_ld_prune_walk) is injected with
LD_PRELOAD, so the real host program runs its real code paths: chromosome runs handed to several device workers, a
relatedness prune chained in front of the LD prune with frozen allele frequencies, and the filtered view feeding the
founder decode.  Expected lists were written by the reference binary for the same command lines.  The product itself
never loads this library; without it (and without a GPU) every device command fails loudly, which is also checked."""
import gzip
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GD = os.path.join(ROOT, "tests", "golden")
BIN = os.path.join(ROOT, "plink_ng_b200", "plink2_b200")


@pytest.fixture(scope="module")
def mock_so(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mock") / "mock_pl2gpu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "harness", "mock_pl2gpu.cc")], check=True)
    return so


def _run(mock_so, args, out, devices=1, log=None):
    env = dict(os.environ, LD_PRELOAD=mock_so, PL2_MOCK_DEVICES=str(devices))
    if log:
        env["PL2_MOCK_LOG"] = log
    r = subprocess.run([BIN] + args + ["--out", out], capture_output=True, text=True, env=env, cwd=GD)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def test_single_worker_ld_prune_matches_reference(mock_so, tmp_path):
    out = str(tmp_path / "o")
    _run(mock_so, ["--bfile", "a", "--indep-pairwise", "50", "5", "0.2"], out)
    assert open(out + ".prune.in", "rb").read() == open(os.path.join(GD, "a_ld.prune.in"), "rb").read()


@pytest.mark.parametrize("gpus,devices", [(1, 1), (3, 3), (8, 2)])
def test_chromosome_runs_over_several_device_workers(mock_so, tmp_path, gpus, devices):
    """Six chromosomes of 120 / 360 / 20 / 1 / 299 / 200 variants: the singleton is never examined, the other five runs are
    taken largest-first by min(--gpus, runs, visible devices) workers, each on its own context, and the merged keep-list
    is the reference's whatever the split."""
    out, log = str(tmp_path / "o"), str(tmp_path / "mock.log")
    stdout = _run(mock_so, ["--bed", "a.bed", "--bim", "a_chr6.bim", "--fam", "a.fam", "--gpus", str(gpus), "--indep-pairwise", "50", "5", "0.2"], out, devices=devices, log=log)
    assert open(out + ".prune.in", "rb").read() == open(os.path.join(GD, "a_chr6.prune.in"), "rb").read()
    calls = [ln.split() for ln in open(log)]
    runs = sorted(int(c[2].split("=")[1]) for c in calls if c[0] == "indep_pairwise")
    assert runs == [20, 120, 200, 299, 360]
    used = {c[1] for c in calls if c[0] == "indep_pairwise"}
    workers = min(gpus, devices, 5)
    assert {c[1] for c in calls if c[0] == "ctx_create"} == {"device=%d" % g for g in range(workers)}
    assert used <= {"device=%d" % g for g in range(workers)} and (workers == 1 or len(used) > 1)
    if workers < gpus:
        assert "Note: --indep-pairwise on %d GPU" % workers in stdout


def test_relatedness_prune_chained_in_front_of_ld_prune(mock_so, tmp_path):
    """--king-cutoff-table leaves 50 founders; the LD prune behind it sees only them but keeps the allele frequencies (and
    so the major alleles / tie-breaks) of all 100 - the reference's own chained run gives the expected list.  The
    50-founder guard is applied before the prune, so the chained run is not refused."""
    (tmp_path / "in.kin0").write_bytes(gzip.open(os.path.join(GD, "a_kingp.kin0.gz"), "rb").read())
    out, log = str(tmp_path / "o"), str(tmp_path / "mock.log")
    stdout = _run(mock_so, ["--bfile", "a", "--king-cutoff-table", str(tmp_path / "in.kin0"), "0.02", "--indep-pairwise", "50", "5", "0.2"], out, log=log)
    assert "50 samples remaining after the relatedness prune." in stdout
    assert open(out + ".prune.in", "rb").read() == open(os.path.join(GD, "g_akct.prune.in"), "rb").read()
    calls = [ln.split()[0] for ln in open(log)]
    assert calls.index("geno_counts") < calls.index("indep_pairwise")  # frequencies frozen from the pre-prune founders first


def test_filtered_view_feeds_the_ld_prune(mock_so, tmp_path):
    out = str(tmp_path / "o")
    _run(mock_so, ["--bfile", "a", "--remove", "x_remove.txt", "--exclude", "x_exclude.txt", "--indep-pairwise", "50", "5", "0.2"], out)
    assert open(out + ".prune.in", "rb").read() == open(os.path.join(GD, "g_afilt.prune.in"), "rb").read()


def test_without_the_stand_in_device_commands_fail_loudly(tmp_path):
    """No GPU in this container and no mock: the product must refuse, not fall back to anything."""
    import shutil

    if shutil.which("nvidia-smi") and subprocess.run(["nvidia-smi", "-L"], capture_output=True).returncode == 0:
        pytest.skip("a GPU is visible")
    r = subprocess.run([BIN, "--bfile", "a", "--indep-pairwise", "50", "5", "0.2", "--out", str(tmp_path / "o")], capture_output=True, text=True, cwd=GD)
    assert r.returncode == 16 and "GPU initialisation failed" in r.stdout


@pytest.mark.parametrize("args,gold", [(["--bfile", "x"], "x.afreq"),
                                       (["--bfile", "x", "--keep", "x_keep1.txt", "x_keep2.txt", "--remove", "x_remove.txt", "--extract", "x_extract.txt", "--exclude", "x_exclude.txt"], "g_xfilt.afreq")])
def test_freq_driver_on_sex_chromosomes_and_filtered_view(mock_so, tmp_path, args, gold):
    """--freq's host side: three counting passes (founders; founder males on chrX; nonfemale founders on chrY) over
    subsets of the view, the reference's ddosage accounting and report format.  With exact counts from the stand-in the
    report is the reference's byte for byte, unfiltered and under the filter fixture."""
    out = str(tmp_path / "o")
    _run(mock_so, args + ["--freq"], out)
    assert open(out + ".afreq", "rb").read() == open(os.path.join(GD, gold), "rb").read()


@pytest.mark.parametrize("args,gold", [(["--bfile", "a", "--r2-unphased"], "a_r2.vcor.gz"),
                                       (["--bfile", "a", "--r2-unphased", "--ld-window", "7", "--ld-window-r2", "0.5"], "a_r2w.vcor.gz"),
                                       (["--bfile", "x", "--not-chr", "X", "--keep", "x_keep1.txt", "x_keep2.txt", "--r2-unphased", "--ld-window-r2", "0.3", "--ld-window-kb", "0.1"], "x_r2.vcor.gz")])
def test_r2_unphased_table_matches_reference(mock_so, tmp_path, args, gold):
    """--r2-unphased: the device screens every pair of the band (here: the stand-in's plain loops behind the same entry
    point, pl2gpu_ld_band_flags), the host recomputes the flagged pairs from bit planes with the reference's arithmetic
    and applies the window / threshold rules.  Tables byte-identical to the reference's: 499,500 candidate pairs of set
    A, a variant-count window, and set X without chrX (female founders missing on chrY, non-founders ignored)."""
    out = str(tmp_path / "o")
    _run(mock_so, args, out)
    assert open(out + ".vcor", "rb").read() == gzip.open(os.path.join(GD, gold), "rb").read()


@pytest.mark.parametrize("args,gold", [(["--bfile", "x", "--keep", "x_keep1.txt", "x_keep2.txt", "--r2-unphased", "--ld-window-r2", "0.1", "--ld-window-kb", "0.05"], "x_r2x.vcor.gz"),
                                       (["--bfile", "x", "--nonfounders", "--r2-unphased", "--ld-window-r2", "0.1", "--chr", "X,Y"], "x_r2nf.vcor.gz")])
def test_r2_unphased_on_chrx_matches_reference(mock_so, tmp_path, args, gold):
    """chrX pairs use the reference's sex-aware statistic (every sum over all founders minus half of the male founders'
    sum, genotypes counted as non-major alleles, fused multiply-adds as in ComputeXR2) and are evaluated on the host for
    every pair of the window - the unweighted device screen is no superset for them.  Tables byte-identical to the
    reference's with males, females, unknown sex and non-founders present, and with --nonfounders frequencies deciding
    the major allele."""
    out = str(tmp_path / "o")
    _run(mock_so, args, out)
    assert open(out + ".vcor", "rb").read() == gzip.open(os.path.join(GD, gold), "rb").read()


def test_r2_unphased_refuses_what_it_does_not_cover(mock_so, tmp_path):
    env = dict(os.environ, LD_PRELOAD=mock_so)
    for args, msg in ((["--bfile", "a", "--r2-unphased", "--ld-window-r2", "0"], "positive --ld-window-r2"), (["--bfile", "a", "--r2-unphased", "square"], "not supported")):
        r = subprocess.run([BIN] + args + ["--out", str(tmp_path / "o")], capture_output=True, text=True, env=env, cwd=GD)
        assert r.returncode != 0 and msg in r.stdout + r.stderr, (args, r.stdout)


def test_nonfounders_frequencies_reach_the_device_commands(mock_so, tmp_path):
    """--nonfounders: the --freq report counts every sample, and the LD prune - whose r^2 still comes from the founders -
    breaks ties with all-sample frequencies (frozen as per-variant overrides by one host counting pass).  Set X has four
    non-founders, enough to change both outputs; expected files are the reference's."""
    out = str(tmp_path / "o")
    stdout = _run(mock_so, ["--bfile", "x", "--nonfounders", "--freq"], out)
    assert "(all samples)" in stdout
    assert open(out + ".afreq", "rb").read() == open(os.path.join(GD, "x_nf.afreq"), "rb").read()
    assert open(out + ".afreq", "rb").read() != open(os.path.join(GD, "x.afreq"), "rb").read()
    _run(mock_so, ["--bfile", "x", "--nonfounders", "--freq", "counts"], out)  # allele dosages: halves for haploid hets on MT
    assert open(out + ".acount", "rb").read() == open(os.path.join(GD, "x_nf.acount"), "rb").read()
    _run(mock_so, ["--bfile", "x", "--chr", "1", "--nonfounders", "--indep-pairwise", "50", "5", "0.2"], out)
    assert open(out + ".prune.in", "rb").read() == open(os.path.join(GD, "x_nf.prune.in"), "rb").read()


def _gold(name):
    p = os.path.join(GD, name)
    return gzip.open(p, "rb").read() if name.endswith(".gz") else open(p, "rb").read()


KING_CASES = [
    (["--bfile", "a", "--make-king-table", "counts", "cols=+ibs1,+ibs", "--make-king", "bin4", "triangle"], {".kin0": "a_king.kin0.gz", ".king.bin": "a_king.king.bin"}),
    (["--bfile", "a", "--make-king-table"], {".kin0": "a_kingp.kin0.gz"}),
    (["--bfile", "a", "--make-king", "square"], {".king": "a_kingsq.king.gz", ".king.id": "a_kingsq.king.id"}),
    (["--bfile", "a", "--make-king-table", "counts", "--king-table-filter", "0.02"], {".kin0": "a_kingfilt.kin0"}),
    (["--bfile", "a", "--make-king-table", "counts", "--parallel", "2", "3"], {".kin0.2": "a_kingpar.kin0.2.gz"}),
    (["--bfile", "q", "--make-king-table", "counts", "cols=+ibs1,+ibs"], {".kin0": "q_king.kin0"}),
    (["--bfile", "x", "--keep", "x_keep1.txt", "x_keep2.txt", "--remove", "x_remove.txt", "--extract", "x_extract.txt", "--exclude", "x_exclude.txt", "--make-king-table"], {".kin0": "g_xfilt.kin0.gz"}),
    (["--bfile", "a", "--gpu-memory", "4", "--make-king-table", "counts", "cols=+ibs1,+ibs", "--make-king", "bin4", "triangle"], {".kin0": "a_king.kin0.gz", ".king.bin": "a_king.king.bin"}),
]


@pytest.mark.parametrize("case", range(len(KING_CASES)))
def test_king_driver_replayed_on_the_cpu(mock_so, tmp_path, case):
    """RunKing around a stand-in KING job (plain-loop pair counts): table / matrix writers, the device-side filter's
    contract, a --parallel piece, the rare-variant NSNP accounting of set Q, a filtered view, and - with the device memory
    capped at 4 MiB - three passes over the variants.  Files byte-identical to the reference's."""
    args, files = KING_CASES[case]
    out = str(tmp_path / "o")
    stdout = _run(mock_so, args, out)
    for ext, gold in files.items():
        assert open(out + ext, "rb").read() == _gold(gold), ext
    if "--gpu-memory" in args:
        assert "3 passes over the variants" in stdout


def test_king_cutoff_chained_into_the_ld_prune(mock_so, tmp_path):
    """`--king-cutoff 0.02 --indep-pairwise 50 5 0.2` in one run, all of it through the host program: KING pass, greedy
    relatedness prune (49 survivors), allele frequencies frozen from the 100 pre-prune founders, survivors dropped from
    the view, LD prune - the reference's chained list.  (The 50-founder guard applies to the pre-prune dataset.)"""
    out, log = str(tmp_path / "o"), str(tmp_path / "mock.log")
    stdout = _run(mock_so, ["--bfile", "a", "--king-cutoff", "0.02", "--indep-pairwise", "50", "5", "0.2"], out, log=log)
    assert "49 samples remaining after the relatedness prune." in stdout
    assert open(out + ".king.cutoff.in.id", "rb").read() == _gold("a_cut.king.cutoff.in.id")
    assert open(out + ".prune.in", "rb").read() == _gold("g_acut.prune.in")
    calls = [ln.split()[0] for ln in open(log)]
    assert calls.index("king_begin") < calls.index("geno_counts") < calls.index("indep_pairwise")


def test_extra_contigs_are_diploid_autosome_like_units(mock_so, tmp_path):
    """--allow-extra-chr: unrecognised contig names (here chrUn_KI270 and GL000.1 carved out of set X) get their own
    codes, are printed as written, stay out of --autosome / numeric --not-chr lists, are kept by KING, and are LD-pruned
    as diploid chromosomes of their own - outputs identical to the reference's; without the flag the file is refused."""
    data = ["--bed", "x.bed", "--bim", "x_contigs.bim", "--fam", "x.fam", "--allow-extra-chr"]
    out = str(tmp_path / "o")
    r = subprocess.run([BIN] + data + ["--not-chr", "1,X", "--make-bed", "--out", out], capture_output=True, text=True, cwd=GD)
    assert r.returncode == 0 and open(out + ".bim", "rb").read() == _gold("x_contigs_sub.bim")
    _run(mock_so, data + ["--not-chr", "X,Y,MT", "--indep-pairwise", "50", "5", "0.2"], out)
    assert open(out + ".prune.in", "rb").read() == _gold("x_contigs.prune.in")
    _run(mock_so, data + ["--make-king-table"], out)
    assert open(out + ".kin0", "rb").read() == _gold("x_contigs.kin0.gz")
    r = subprocess.run([BIN] + data[:-1] + ["--make-bed", "--out", out], capture_output=True, text=True, cwd=GD)
    assert r.returncode != 0 and "--allow-extra-chr" in r.stdout


def _f32_close(path, gold):
    import numpy as np

    got = np.fromfile(path, dtype=np.float32)
    ref = np.frombuffer(_gold(gold), dtype=np.float32)
    assert got.shape == ref.shape
    assert np.all(np.abs(got.astype(np.float64) - ref.astype(np.float64)) <= 1.2e-7 * np.abs(ref) + 5e-10)


def _text_close(path, gold, rtol=1.2e-5, atol=1e-9):
    got = open(path).read().split("\n")
    ref = _gold(gold).decode().split("\n")
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        if a != b:
            ta, tb = a.split("\t"), b.split("\t")
            assert len(ta) == len(tb)
            for x, y in zip(ta, tb):
                assert x == y or abs(float(x) - float(y)) <= rtol * abs(float(y)) + atol, (a, b)


def test_grm_driver_and_writers_replayed_on_the_cpu(mock_so, tmp_path):
    """RunGrm around a stand-in GRM job (plain fp64 loops): every output form of the relationship matrix against the
    reference's files - .grm.bin / .grm.N.bin / .grm.id, the text list, the sparse list, --make-rel cov bin4 and square
    text, meanimpute, and --read-freq frequencies reaching the standardisation."""
    out = str(tmp_path / "o")
    _run(mock_so, ["--bfile", "a", "--make-grm-bin"], out)
    _f32_close(out + ".grm.bin", "a_grm.grm.bin")
    assert open(out + ".grm.N.bin", "rb").read() == _gold("a_grm.grm.N.bin") and open(out + ".grm.id", "rb").read() == _gold("a_grm.grm.id")
    _run(mock_so, ["--bfile", "a", "--make-grm-list"], out)
    _text_close(out + ".grm", "a_grml.grm.gz")
    _run(mock_so, ["--bfile", "a", "--make-grm-sparse", "0.02"], out)
    got = {tuple(ln.split("\t")[:2]): float(ln.split("\t")[2]) for ln in open(out + ".grm.sp").read().split("\n") if ln}
    ref = {tuple(ln.split("\t")[:2]): float(ln.split("\t")[2]) for ln in _gold("a_grmsp.grm.sp").decode().split("\n") if ln}
    assert all(abs(got.get(k, ref.get(k)) - 0.02) < 1e-8 for k in set(got) ^ set(ref))
    assert all(abs(got[k] - ref[k]) <= 2e-9 + 1.5e-8 * abs(ref[k]) for k in set(got) & set(ref)) and len(ref) == 1380
    _run(mock_so, ["--bfile", "a", "--make-rel", "cov", "bin4", "triangle"], out)
    _f32_close(out + ".rel.bin", "a_relcov.rel.bin")
    _run(mock_so, ["--bfile", "a", "--make-rel", "square"], out)
    _text_close(out + ".rel", "a_rel.rel.gz")
    _run(mock_so, ["--bfile", "a", "--make-grm-bin", "meanimpute"], out)
    _f32_close(out + ".grm.bin", "a_grmmi.grm.bin")
    _run(mock_so, ["--bfile", "a", "--read-freq", "a_rf.afreq", "--make-grm-bin"], out)
    _f32_close(out + ".grm.bin", "a_rf.grm.bin")


def test_exact_pca_driver_and_prune_chaining_replayed_on_the_cpu(mock_so, tmp_path):
    """Exact --pca on the stand-in's eigen-solver (eigenvalues + eigenvectors up to sign vs the reference), then the two
    chained forms also checked through the device (tests/test_filters_gpu.py): --king-cutoff -> --make-grm-bin and --king-cutoff-table -> --pca, both with
    the pre-prune allele frequencies."""
    import numpy as np

    out = str(tmp_path / "o")
    _run(mock_so, ["--bfile", "a", "--pca", "4"], out)
    assert np.allclose(np.loadtxt(out + ".eigenval"), np.loadtxt(os.path.join(GD, "a_pca.eigenval")), rtol=2e-5)
    got = np.loadtxt(out + ".eigenvec", skiprows=1, usecols=(2, 3, 4, 5))
    want = np.loadtxt(os.path.join(GD, "a_pca.eigenvec"), skiprows=1, usecols=(2, 3, 4, 5))
    assert np.allclose(got * np.sign((got * want).sum(axis=0)), want, atol=2e-5)
    _run(mock_so, ["--bfile", "a", "--king-cutoff", "0.02", "--make-grm-bin"], out)
    _f32_close(out + ".grm.bin", "g_acut.grm.bin")
    (tmp_path / "in.kin0").write_bytes(_gold("a_kingp.kin0.gz"))
    _run(mock_so, ["--bfile", "a", "--king-cutoff-table", str(tmp_path / "in.kin0"), "0.02", "--pca", "3"], out)
    assert np.allclose(np.loadtxt(out + ".eigenval"), np.loadtxt(os.path.join(GD, "g_akct.eigenval")), rtol=2e-5)
    got = np.loadtxt(out + ".eigenvec", skiprows=1, usecols=(2, 3, 4))
    want = np.loadtxt(os.path.join(GD, "g_akct.eigenvec"), skiprows=1, usecols=(2, 3, 4))
    assert got.shape == want.shape == (50, 3) and np.allclose(got * np.sign((got * want).sum(axis=0)), want, atol=2e-5)


SCORE_CASES = [(("header",), "a_sc.sscore"), (("header", "no-mean-imputation", "cols=+scoresums,+denom"), "a_sc2.sscore"), (("header", "center", "cols=+scoresums"), "a_sc_center.sscore"),
               (("header", "variance-standardize", "cols=+scoresums"), "a_sc_varstd.sscore"), (("header", "dominant", "list-variants", "cols=+scoresums,+denom"), "a_sc_dominant.sscore"),
               (("header", "recessive", "cols=+scoresums,+denom"), "a_sc_recessive.sscore")]


@pytest.mark.parametrize("flags,gold", SCORE_CASES)
def test_score_driver_replayed_on_the_cpu(mock_so, tmp_path, flags, gold):
    """RunScore (file parsing, allele matching, mean-imputation / centering / dominance weight tables, report columns)
    around a stand-in accumulator: the reference's .sscore reports, integer columns exactly and averages / sums to the
    printed digits."""
    out = str(tmp_path / "o")
    stdout = _run(mock_so, ["--bfile", "a", "--score", "a_score.txt"] + list(flags), out)
    assert "400 variants processed" in stdout and "7 were skipped due to mismatching allele codes" in stdout
    _text_close(out + ".sscore", gold, rtol=2e-5, atol=2e-9)
    if "list-variants" in flags:
        assert open(out + ".sscore.vars", "rb").read() == _gold("a_sc.sscore.vars")


def test_score_after_a_relatedness_prune_uses_frozen_frequencies(mock_so, tmp_path):
    out = str(tmp_path / "o")
    _run(mock_so, ["--bfile", "a", "--king-cutoff", "0.02", "--score", "a_score.txt", "header", "cols=+scoresums,+denom"], out)
    _text_close(out + ".sscore", "g_acut.sscore", rtol=2e-5, atol=2e-9)


def test_pair_list_king_and_variant_score_drivers_replayed_on_the_cpu(mock_so, tmp_path):
    """The remaining device-backed drivers: pair-list KING (--king-table-subset with the reference's own table as the
    list + threshold, an IID-only list, rel-check's natural-sort pair lists on two fixtures) and --variant-score (weights
    file parsing, per-variant sums, report columns) - files as the reference wrote them."""
    out = str(tmp_path / "o")
    (tmp_path / "in.kin0").write_bytes(_gold("a_kingp.kin0.gz"))
    _run(mock_so, ["--bfile", "a", "--make-king-table", "counts", "--king-table-subset", str(tmp_path / "in.kin0"), "-0.05"], out)
    assert open(out + ".kin0", "rb").read() == _gold("a_kingsub.kin0.gz")
    _run(mock_so, ["--bfile", "a", "--make-king-table", "counts", "cols=+ibs1", "--king-table-subset", "a_sub2.txt"], out)
    assert open(out + ".kin0", "rb").read() == _gold("a_kingsub2.kin0")
    _run(mock_so, ["--bfile", "r", "--make-king-table", "rel-check", "counts"], out)
    assert open(out + ".kin0", "rb").read() == _gold("r_relcheck.kin0")
    _run(mock_so, ["--bfile", "s", "--make-king-table", "rel-check"], out)
    assert open(out + ".kin0", "rb").read() == _gold("s_relcheck.kin0.gz")
    _run(mock_so, ["--bfile", "a", "--variant-score", "a_vscore_weights.txt"], out)
    _text_close(out + ".vscore", "a_vs.vscore", rtol=2e-5, atol=1e-9)
    _run(mock_so, ["--bfile", "a", "--variant-score", "a_vscore_weights.txt", "cols=+altfreq"], out)
    _text_close(out + ".vscore", "a_vs_altfreq.vscore", rtol=2e-5, atol=1e-9)


@pytest.fixture(scope="module")
def synth_1600(tmp_path_factory):
    """1,600 samples x 200 variants: enough rows for three devices at the drivers' minimum of 512 rows per device."""
    import sys

    sys.path.insert(0, ROOT)
    from oracle import synth

    prefix = str(tmp_path_factory.mktemp("s1600") / "s")
    synth.write_bed(prefix, 1600, 200, seed=3)
    return prefix


MULTI_GPU_RUNS = [
    (["--make-king-table", "counts", "--make-king", "bin4", "triangle"], (".kin0", ".king.bin", ".king.id"), "king_begin"),
    (["--make-king-table", "counts", "--king-table-filter", "0.01"], (".kin0",), "king_begin"),
    (["--make-grm-bin"], (".grm.bin", ".grm.N.bin", ".grm.id"), "grm_begin"),
]


@pytest.mark.parametrize("gpus", [2, 3])
@pytest.mark.parametrize("run", range(len(MULTI_GPU_RUNS)))
def test_gpus_split_matches_one_device(mock_so, synth_1600, tmp_path, run, gpus):
    """--gpus: the KING and GRM drivers cut the triangle into one row slab per device and hand each device its slice of
    every decoded block (topped up with all-missing rows to a multiple of the device count); the stand-in all-gathers
    the slices like NCCL.  Files byte-identical to the one-device run, with more than one device holding a job."""
    args, exts, begin = MULTI_GPU_RUNS[run]
    one, many, log = str(tmp_path / "one"), str(tmp_path / "many"), str(tmp_path / "mock.log")
    _run(mock_so, ["--bfile", synth_1600] + args, one)
    stdout = _run(mock_so, ["--bfile", synth_1600] + args + ["--gpus", str(gpus)], many, devices=3, log=log)
    assert "reduced" not in stdout and "computed on" not in stdout
    for ext in exts:
        assert open(many + ext, "rb").read() == open(one + ext, "rb").read(), ext
    began = {ln.split()[1] for ln in open(log) if ln.split()[0] == begin}
    assert began == {"device=%d" % g for g in range(gpus)}
