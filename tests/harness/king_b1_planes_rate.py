"""Default KING kernel time of several builds of libpl2gpu.so, alternating in one session, on one GPU.

Each build is a library file; every measurement runs in a fresh process that imports the package from a temporary
copy with that library in place, so the builds never share a process.  For each shape (default 16,384 x 65,536 and
60,000 x 131,072) and repetition the builds take turns: one job per process, `--warmup` launches of the whole
random block, then `--launches` timed ones, each timed with the CUDA events the library records around its tensor
kernel launches (pl2gpu_king_last_kernel_ms).  With `--profile` each build instead runs once under torch.profiler
(CUDA activities) and reports the device time per block of the re-tiling kernel on the prep stream
(geno_tile_rows_kernel) and of the KING kernels.  The card name and power limit, and the SM clock and power draw
sampled with nvidia-smi during the timed launches, are printed beside every number.

    python tests/harness/king_b1_planes_rate.py --lib parent=/path/plink_ng_b200/libpl2gpu.so --lib control=/path/b.so \\
        --lib cluster=plink_ng_b200/libpl2gpu.so [--reps 2] [--out DIR/planes_rate.json]

A library that sits in a package directory is loaded with that package's Python bindings (a build with another
ABI); any other library with this tree's.  Comparing the plane-copy kernel with and without row-tile pairs needs a
build whose tile list has no pairs (every tile then runs without a partner): the same sources with BuildTileList's
`row_pairs` argument false in KingBegin.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def child(lib, n, m, warmup, launches, profile=False):
    tmp = tempfile.mkdtemp(prefix="kb1_rate_")
    try:
        pkg = os.path.join(tmp, "plink_ng_b200")
        os.makedirs(pkg)
        # the Python bindings that go with the library: those next to it (a whole package of another build), else this tree's
        src = os.path.dirname(lib) if os.path.exists(os.path.join(os.path.dirname(lib), "capi.py")) else os.path.join(ROOT, "plink_ng_b200")
        for f in os.listdir(src):
            if f.endswith(".py"):
                shutil.copy(os.path.join(src, f), pkg)
        shutil.copy(lib, os.path.join(pkg, "libpl2gpu.so"))
        sys.path.insert(0, tmp)
        import numpy as np

        import plink_ng_b200 as p
        from plink_ng_b200.host import KING_ALGO_TENSOR_TS, KingJob

        # random 2-bit codes (a quarter missing), packed as PgrGet rows
        packed = np.random.default_rng(1).integers(0, 2**63, size=(m, -(-n // 32)), dtype=np.uint64)
        clocks, stop = [], threading.Event()

        def sample():
            while not stop.wait(0.25):
                clocks.append(smi("clocks.sm,power.draw"))

        with p.GpuContext(0) as ctx, KingJob(ctx, n, 0, n, KING_ALGO_TENSOR_TS, m) as job:
            for _ in range(warmup):
                job.add_variants(packed)
                job.last_kernel_ms()
            th = threading.Thread(target=sample)
            th.start()
            ms, prof = [], None
            if profile:
                import torch

                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(launches):
                        job.add_variants(packed)
                        ms.append(job.last_kernel_ms())
                    torch.cuda.synchronize()
            else:
                for _ in range(launches):
                    job.add_variants(packed)
                    ms.append(job.last_kernel_ms())
            stop.set()
            th.join()
        kernels = {}
        if prof is not None:
            for e in prof.key_averages():
                if "geno_tile_rows_kernel" in e.key or "king_b1_kernel" in e.key:
                    t = getattr(e, "device_time_total", None)
                    t = e.cuda_time_total if t is None else t
                    kernels[e.key] = {"calls": e.count, "ms_per_block": round(t / 1e3 / launches, 3)}
        print(json.dumps({"kernel_ms": ms, "sm_clock_power": clocks, "profile": kernels}))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="name=path of a libpl2gpu.so build")
    ap.add_argument("--shape", action="append", default=[], help="samples,variants (default: 16384,65536 and 60000,131072)")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--launches", type=int, default=0, help="timed launches per process (default: 20 below 30,000 samples, else 4)")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", nargs=6, metavar=("LIB", "N", "M", "WARMUP", "LAUNCHES", "PROFILE"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        lib, n, m, w, k, prof = args.child
        child(lib, int(n), int(m), int(w), int(k), prof == "1")
        return

    libs = [s.split("=", 1) for s in args.lib]
    shapes = [tuple(int(x) for x in s.split(",")) for s in args.shape] or [(16384, 65536), (60000, 131072)]
    card = smi("name,power.limit,clocks.max.sm")
    res = {"card (name, power limit, max SM clock)": card, "runs": []}
    print(f"card: {card}", flush=True)
    for n, m in shapes:
        launches = args.launches or (20 if n < 30000 else 4)
        for rep in range(1 if args.profile else args.reps):
            for name, lib in libs:
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", os.path.abspath(lib), str(n), str(m), str(args.warmup), str(launches), "1" if args.profile else "0"], capture_output=True, text=True)
                if out.returncode:
                    raise SystemExit(f"{name} at {n} x {m} failed:\n{out.stdout}\n{out.stderr}")
                r = json.loads(out.stdout.strip().splitlines()[-1])
                ms = sorted(r["kernel_ms"])
                row = {"build": name, "samples": n, "variants": m, "rep": rep, "kernel_ms_min": round(ms[0], 3), "kernel_ms_median": round(ms[len(ms) // 2], 3),
                       "kernel_ms_max": round(ms[-1], 3), "card": card, "sm_clock_power": r["sm_clock_power"][-3:], "profile": r["profile"]}
                res["runs"].append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
