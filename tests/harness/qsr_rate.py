"""Device time of `--q-score-range` scoring against one plain `--score` pass, on one GPU.

For 60,000 samples x 131,072 scored entries (eight staging batches of 16,384), genotypes resident on the device, it
times whole add calls with CUDA events on the library's stream (each call ends in a stream synchronise), for 1 and 4
coefficient columns:
  plain     pl2gpu_score_begin_cols + pl2gpu_score_add_variants (one pass of plain --score);
  nested    pl2gpu_score_begin_classes + _add_variants_classes with 8 nested ranges (p <= 1e-5 .. p <= 1; the entries
            split into 8 classes of growing size);
  disjoint  the same with 8 disjoint ranges of equal width (8 classes of equal size).
The entries' p-values are uniform and in random order, so every staging batch holds every class in many pieces.  The
first call of every shape is a warm-up.  Legs alternate within each round.

    python tests/harness/qsr_rate.py [--rounds 3] [--reps 5] [--out DIR/qsr_rate.json]

The card name and power limit are read with nvidia-smi in the same run and printed beside the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
LIB = os.path.join(ROOT, "plink_ng_b200", "libpl2gpu.so")
SAMPLES, ENTRIES = 60000, 131072
NESTED = [1e-5, 1e-4, 1e-3, 1e-2, 0.05, 0.1, 0.5, 1.0]  # upper bounds, lower bound 0


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return out.strip().splitlines()[0]


def classes_of(p, form):
    """The class of each entry: the set of ranges its p-value lies in, numbered in first appearance (as the host does)."""
    import numpy as np

    if form == "nested":
        member = p[:, None] <= np.array(NESTED)[None, :]
    else:
        edges = np.linspace(0.0, 1.0, 9)
        member = (p[:, None] >= edges[None, :-1]) & (p[:, None] <= edges[None, 1:])
    keys, cls = np.unique(member, axis=0, return_inverse=True)
    return cls.astype(np.uint32).ravel(), len(keys)


def main():
    import numpy as np
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
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
    lib.pl2gpu_score_end.argtypes = [vp]
    lib.pl2gpu_last_error.restype = C.c_char_p

    def check(rc, what):
        if rc:
            raise RuntimeError(f"{what}: {lib.pl2gpu_last_error().decode()}")

    ctx = C.c_void_p()
    check(lib.pl2gpu_ctx_create(0, C.byref(ctx)), "pl2gpu_ctx_create")
    row_bytes = (SAMPLES + 31) // 32 * 8
    g = torch.randint(0, 256, (ENTRIES, row_bytes), dtype=torch.uint8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    torch.cuda.synchronize()
    d4 = np.full(ENTRIES, 0x24, dtype=np.uint8)
    p = np.random.default_rng(7).random(ENTRIES)
    forms = {"nested": classes_of(p, "nested"), "disjoint": classes_of(p, "disjoint")}
    print("classes:", {k: v[1] for k, v in forms.items()}, flush=True)

    def leg(form, sc, w4):
        h = C.c_void_p()
        if form == "plain":
            check(lib.pl2gpu_score_begin_cols(ctx, SAMPLES, sc, C.byref(h)), "pl2gpu_score_begin_cols")
        else:
            check(lib.pl2gpu_score_begin_classes(ctx, SAMPLES, sc, forms[form][1], C.byref(h)), "pl2gpu_score_begin_classes")
        times = []
        try:
            for r in range(a.reps + 1):
                check(lib.pl2gpu_ctx_event_record(ctx, 0), "event")
                if form == "plain":
                    check(lib.pl2gpu_score_add_variants(h, C.c_void_p(g.data_ptr()), row_bytes, ENTRIES, 1, w4.ctypes.data, d4.ctypes.data), "pl2gpu_score_add_variants")
                else:
                    cls = forms[form][0]
                    check(lib.pl2gpu_score_add_variants_classes(h, C.c_void_p(g.data_ptr()), row_bytes, ENTRIES, 1, cls.ctypes.data, None, w4.ctypes.data, None, d4.ctypes.data), "pl2gpu_score_add_variants_classes")
                check(lib.pl2gpu_ctx_event_record(ctx, 1), "event")
                ms = C.c_float()
                check(lib.pl2gpu_ctx_event_elapsed_ms(ctx, 0, 1, C.byref(ms)), "elapsed")
                if r:  # the first call is the warm-up
                    times.append(ms.value)
        finally:
            lib.pl2gpu_score_end(h)
        return times

    runs = []
    legs = [("plain", 1), ("nested", 1), ("disjoint", 1), ("plain", 4), ("nested", 4), ("disjoint", 4)]
    weights = {sc: np.random.default_rng(sc).normal(size=(ENTRIES, sc, 4)) for sc in (1, 4)}
    for rnd in range(a.rounds):
        for form, sc in legs if rnd % 2 == 0 else legs[::-1]:
            t = leg(form, sc, weights[sc])
            runs.append({"form": form, "score_ct": sc, "round": rnd, "ms": t})
            print(form, sc, rnd, "%.2f - %.2f ms" % (min(t), max(t)), flush=True)
    summary = {}
    for run in runs:
        summary.setdefault((run["form"], run["score_ct"]), []).extend(run["ms"])
    for (form, sc), v in sorted(summary.items(), key=lambda kv: (kv[0][1], kv[0][0])):
        med = sorted(v)[len(v) // 2]
        plain = sorted(summary[("plain", sc)])[len(summary[("plain", sc)]) // 2]
        print(f"{form} score_ct={sc}: min {min(v):.2f} ms, median {med:.2f} ms, max {max(v):.2f} ms over {len(v)} calls; median / plain {med / plain:.2f} ({SAMPLES} samples x {ENTRIES} entries)")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": info, "samples": SAMPLES, "entries": ENTRIES, "classes": {k: v[1] for k, v in forms.items()}, "runs": runs}, f, indent=1)


if __name__ == "__main__":
    main()
