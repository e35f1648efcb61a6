"""Device time of the `--score` accumulation for several coefficient columns in one pass, on one GPU.

For 60,000 samples x 131,072 scored entries (eight staging batches of 16,384), genotypes resident on the device, it
times whole pl2gpu_score_add_variants calls with CUDA events on the library's stream (the call ends in a stream
synchronise) for score_ct = 1, 4, 16 and 64 columns, after one warm-up call per shape.  With --parent-lib it also
times score_ct = 1 through another build of the library (e.g. the parent commit's), in separate processes that
alternate with this tree's, so both are measured in the same session.

    python tests/harness/score_cols_rate.py [--parent-lib PATH] [--rounds 3] [--out DIR/score_cols_rate.json]

The card name and power limit are read with nvidia-smi in the same run and printed beside the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
LIB = os.path.join(ROOT, "plink_ng_b200", "libpl2gpu.so")
SAMPLES, ENTRIES = 60000, 131072


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return out.strip().splitlines()[0]


def worker(lib_path, cols, reps):
    import numpy as np
    import torch

    lib = C.CDLL(lib_path)
    vp = C.c_void_p
    lib.pl2gpu_ctx_create.argtypes = [C.c_int, vp]
    lib.pl2gpu_ctx_event_record.argtypes = [vp, C.c_int]
    lib.pl2gpu_ctx_event_elapsed_ms.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_float)]
    lib.pl2gpu_score_begin.argtypes = [vp, C.c_uint32, vp]
    lib.pl2gpu_score_add_variants.argtypes = [vp, vp, C.c_uint64, C.c_uint32, C.c_int, vp, vp]
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
    res = {}
    for sc in cols:
        w4 = np.random.default_rng(sc).normal(size=(ENTRIES, sc, 4))
        h = C.c_void_p()
        if sc == 1:
            check(lib.pl2gpu_score_begin(ctx, SAMPLES, C.byref(h)), "pl2gpu_score_begin")
        else:
            lib.pl2gpu_score_begin_cols.argtypes = [vp, C.c_uint32, C.c_uint32, vp]
            check(lib.pl2gpu_score_begin_cols(ctx, SAMPLES, sc, C.byref(h)), "pl2gpu_score_begin_cols")
        times = []
        try:
            for r in range(reps + 1):
                check(lib.pl2gpu_ctx_event_record(ctx, 0), "event")
                check(lib.pl2gpu_score_add_variants(h, C.c_void_p(g.data_ptr()), row_bytes, ENTRIES, 1, w4.ctypes.data, d4.ctypes.data), "pl2gpu_score_add_variants")
                check(lib.pl2gpu_ctx_event_record(ctx, 1), "event")
                ms = C.c_float()
                check(lib.pl2gpu_ctx_event_elapsed_ms(ctx, 0, 1, C.byref(ms)), "elapsed")
                if r:  # the first call is the warm-up
                    times.append(ms.value)
        finally:
            lib.pl2gpu_score_end(h)
        res[sc] = times
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", nargs=2, default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.worker[0], [int(x) for x in a.worker[1].split(",")], a.reps)
        return
    info = card()
    print("card, power limit, max SM clock:", info, flush=True)
    runs = []
    for rnd in range(a.rounds):
        legs = [("tree", LIB, "1,4,16,64")] + ([("parent", a.parent_lib, "1")] if a.parent_lib else [])
        for name, path, cols in legs if rnd % 2 == 0 else legs[::-1]:
            out = subprocess.run([sys.executable, __file__, "--reps", str(a.reps), "--worker", path, cols], capture_output=True, text=True, check=True).stdout
            r = json.loads(out.strip().splitlines()[-1])
            runs.append({"build": name, "round": rnd, "ms": r})
            print(name, rnd, {k: "%.2f - %.2f ms" % (min(v), max(v)) for k, v in r.items()}, flush=True)
    summary = {}
    for build in ("tree", "parent"):
        for run in runs:
            if run["build"] == build:
                for k, v in run["ms"].items():
                    summary.setdefault(f"{build} score_ct={k}", []).extend(v)
    for k, v in summary.items():
        print(f"{k}: min {min(v):.2f} ms, median {sorted(v)[len(v) // 2]:.2f} ms, max {max(v):.2f} ms over {len(v)} calls ({SAMPLES} samples x {ENTRIES} entries)")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": info, "samples": SAMPLES, "entries": ENTRIES, "runs": runs}, f, indent=1)


if __name__ == "__main__":
    main()
