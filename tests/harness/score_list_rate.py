"""Device time of `--score-list` scoring (pl2gpu_score_add_entries) against its alternatives, on one GPU.

60,000 samples, one coefficient column, genotypes in pinned host memory (as the host program streams them) and
added in calls of 16,384 staged rows.  Two list shapes:
  chr22    22 disjoint files of 4,096 variants each (per-chromosome files): 90,112 rows, one entry each;
  overlap  8 files over 16,384 variants, each naming a variant with probability 3/4: about 98,000 entries.
Legs, timed with CUDA events on the library's stream around the add calls only (each call ends in a stream synchronise):
  entries   one job of one class per file, each variant staged once, pl2gpu_score_add_entries;
  per_file  one plain job per file (pl2gpu_score_begin_cols + _add_variants), i.e. one --score pass per file;
  dup_rows  one job of one class per file, the rows duplicated once per entry on the host and added with
            pl2gpu_score_add_variants_classes.
Next to each time it prints the host-to-device bytes the leg copies (genotype rows, weight tables, named-allele
dosages and the gather order).  The first call of every leg is a warm-up; legs alternate within each round.

    python tests/harness/score_list_rate.py [--rounds 2] [--reps 3] [--out DIR/score_list_rate.json]

The card name and power limit are read with nvidia-smi in the same run and printed beside the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
LIB = os.path.join(ROOT, "plink_ng_b200", "libpl2gpu.so")
SAMPLES, BATCH = 60000, 16384


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return out.strip().splitlines()[0]


def shapes():
    """{shape: (row_ct, per-file sorted row lists)}."""
    import numpy as np

    rng = np.random.default_rng(3)
    chr22 = [np.arange(k * 4096, (k + 1) * 4096, dtype=np.uint32) for k in range(22)]
    overlap = [np.flatnonzero(rng.random(16384) < 0.75).astype(np.uint32) for _ in range(8)]
    return {"chr22": (22 * 4096, chr22), "overlap": (16384, overlap)}


def main():
    import numpy as np
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    print("card, power limit, max SM clock:", info, flush=True)
    lib = C.CDLL(LIB)
    vp = C.c_void_p
    lib.pl2gpu_ctx_create.argtypes = [C.c_int, vp]
    lib.pl2gpu_ctx_event_record.argtypes = [vp, C.c_int]
    lib.pl2gpu_ctx_event_elapsed_ms.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_float)]
    lib.pl2gpu_score_begin_cols.argtypes = [vp, C.c_uint32, C.c_uint32, vp]
    lib.pl2gpu_score_begin_classes.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, vp]
    lib.pl2gpu_score_add_variants.argtypes = [vp, vp, C.c_uint64, C.c_uint32, C.c_int, vp, vp]
    lib.pl2gpu_score_add_variants_classes.argtypes = [vp, vp, C.c_uint64, C.c_uint32, C.c_int, vp, vp, vp, vp, vp]
    lib.pl2gpu_score_add_entries.argtypes = [vp, vp, C.c_uint64, C.c_uint32, C.c_int, C.c_uint32, vp, vp, vp, vp, vp, vp]
    lib.pl2gpu_score_end.argtypes = [vp]
    lib.pl2gpu_last_error.restype = C.c_char_p

    def check(rc, what):
        if rc:
            raise RuntimeError(f"{what}: {lib.pl2gpu_last_error().decode()}")

    ctx = C.c_void_p()
    check(lib.pl2gpu_ctx_create(0, C.byref(ctx)), "pl2gpu_ctx_create")
    row_bytes = (SAMPLES + 31) // 32 * 8
    gen = torch.Generator().manual_seed(5)

    def pinned_rows(ct):
        t = torch.randint(0, 256, (ct, row_bytes), dtype=torch.uint8, generator=gen).pin_memory()
        return t, t.data_ptr()

    def timed(fn):
        check(lib.pl2gpu_ctx_event_record(ctx, 0), "event")
        fn()
        check(lib.pl2gpu_ctx_event_record(ctx, 1), "event")
        ms = C.c_float()
        check(lib.pl2gpu_ctx_event_elapsed_ms(ctx, 0, 1, C.byref(ms)), "elapsed")
        return ms.value

    runs, summary = [], {}
    for shape, (row_ct, files) in shapes().items():
        F = len(files)
        rows_t, rows_p = pinned_rows(row_ct)
        # entries in row order, one class per file; a row's entries in list order
        er = np.concatenate(files)
        ec = np.concatenate([np.full(len(f), k, dtype=np.uint32) for k, f in enumerate(files)])
        order = np.argsort(er, kind="stable")
        er, ec = np.ascontiguousarray(er[order]), np.ascontiguousarray(ec[order])
        E = er.size
        w4 = np.random.default_rng(1).normal(size=(E, 1, 4))
        d4 = np.full(E, 0x24, dtype=np.uint8)
        dup_t = torch.from_numpy(rows_t.numpy()[er]).pin_memory()
        per_file_rows = [torch.from_numpy(rows_t.numpy()[f]).pin_memory() for f in files]
        per_file_w = [np.ascontiguousarray(w4[ec == k]) for k in range(F)]
        print(f"{shape}: {F} files, {row_ct} rows, {E} entries", flush=True)

        def entries_leg():
            h = C.c_void_p()
            check(lib.pl2gpu_score_begin_classes(ctx, SAMPLES, 1, F, C.byref(h)), "begin_classes")
            try:
                def run():
                    for r0 in range(0, row_ct, BATCH):
                        cnt = min(BATCH, row_ct - r0)
                        e0, e1 = np.searchsorted(er, r0), np.searchsorted(er, r0 + cnt)
                        rows = np.ascontiguousarray(er[e0:e1] - r0)
                        check(lib.pl2gpu_score_add_entries(h, rows_p + r0 * row_bytes, row_bytes, cnt, 0, int(e1 - e0), rows.ctypes.data, ec[e0:].ctypes.data, None, w4[e0:].ctypes.data, None, d4[e0:].ctypes.data), "add_entries")
                return timed(run)
            finally:
                lib.pl2gpu_score_end(h)

        def per_file_leg():
            def run():
                for k in range(F):
                    h = C.c_void_p()
                    check(lib.pl2gpu_score_begin_cols(ctx, SAMPLES, 1, C.byref(h)), "begin_cols")
                    try:
                        t, w = per_file_rows[k], per_file_w[k]
                        for r0 in range(0, t.shape[0], BATCH):
                            cnt = min(BATCH, t.shape[0] - r0)
                            check(lib.pl2gpu_score_add_variants(h, t.data_ptr() + r0 * row_bytes, row_bytes, cnt, 0, w[r0:].ctypes.data, d4.ctypes.data), "add_variants")
                    finally:
                        lib.pl2gpu_score_end(h)
            return timed(run)

        def dup_leg():
            h = C.c_void_p()
            check(lib.pl2gpu_score_begin_classes(ctx, SAMPLES, 1, F, C.byref(h)), "begin_classes")
            try:
                def run():
                    for e0 in range(0, E, BATCH):
                        cnt = min(BATCH, E - e0)
                        check(lib.pl2gpu_score_add_variants_classes(h, dup_t.data_ptr() + e0 * row_bytes, row_bytes, cnt, 0, ec[e0:].ctypes.data, None, w4[e0:].ctypes.data, None, d4[e0:].ctypes.data), "add_variants_classes")
                return timed(run)
            finally:
                lib.pl2gpu_score_end(h)

        table = 33  # bytes per entry: four fp64 weights and the named-allele dosage byte
        h2d = {"entries": row_ct * row_bytes + E * (table + 4), "per_file": E * (row_bytes + table), "dup_rows": E * (row_bytes + table + 4)}
        legs = {"entries": entries_leg, "per_file": per_file_leg, "dup_rows": dup_leg}
        for leg in legs.values():
            leg()  # warm-up
        for rnd in range(a.rounds):
            for name in (list(legs) if rnd % 2 == 0 else list(legs)[::-1]):
                t = [legs[name]() for _ in range(a.reps)]
                runs.append({"shape": shape, "leg": name, "round": rnd, "ms": t, "h2d_bytes": h2d[name]})
                summary.setdefault((shape, name), []).extend(t)
                print(shape, name, rnd, "%.2f - %.2f ms" % (min(t), max(t)), flush=True)
        for name in legs:
            v = sorted(summary[(shape, name)])
            base = sorted(summary[(shape, "entries")])[len(v) // 2]
            print(f"{shape} {name}: median {v[len(v) // 2]:.2f} ms (min {v[0]:.2f}, max {v[-1]:.2f}, {len(v)} calls), / entries {v[len(v) // 2] / base:.2f}, H2D {h2d[name] / 1e9:.3f} GB", flush=True)
        del rows_t, dup_t, per_file_rows
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": info, "samples": SAMPLES, "runs": runs}, f, indent=1)


if __name__ == "__main__":
    main()
