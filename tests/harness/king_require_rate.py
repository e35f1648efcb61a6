"""Device time of the three ways to get the `--king-table-require` pairs, on one GPU.

For N samples x M variants (random codes) and r = 1 %, 5 % and 20 % of N required samples it times, with a host clock
around work that ends in a device synchronise:
  - dense: the mapped job (pl2gpu_king_begin_mapped) over rows [N - r, N) with the required samples last, plus the
    read-back of all its counts;
  - full:  the full-triangle job (pl2gpu_king_begin_ex, rows [0, N)), without read-back (it would not fit the host);
  - list:  the pair-list kernel (pl2gpu_king_pairs_begin) on the same r x N pairs, plus its read-back, only where the
    list has at most --max-list-pairs pairs (its traffic grows as pairs x M).
The variants go in as the same 65,536-variant block repeated M / 65,536 times.  One warm-up job per shape is run first.

    python tests/harness/king_require_rate.py [--samples 16384 60000] [--variants 131072] [--out DIR/king_require_rate.json]

The card name and power limit are read with nvidia-smi in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, nargs="+", default=[16384, 60000])
    ap.add_argument("--variants", type=int, default=131072)
    ap.add_argument("--fractions", type=float, nargs="+", default=[0.01, 0.05, 0.20])
    ap.add_argument("--max-list-pairs", type=int, default=20_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np

    import plink_ng_b200 as p
    from plink_ng_b200.host import KingJob, KingPairJob, MappedKingJob

    block = 65536
    reps = max(1, args.variants // block)
    res = {"card": card(), "variants": reps * block, "runs": []}
    rng = np.random.default_rng(1)
    with p.GpuContext(0) as ctx:

        def timed(make, readback):
            t0 = time.perf_counter()
            with make() as job:
                for _ in range(reps):
                    job.add_variants(packed)
                ctx.synchronize()
                t1 = time.perf_counter()
                if readback:
                    job.counts()
                t2 = time.perf_counter()
            return round(t1 - t0, 3), round(t2 - t1, 3)

        for n in args.samples:
            words = (n + 31) // 32
            packed = rng.integers(0, 2**63, size=(block, words), dtype=np.uint64)
            with MappedKingJob(ctx, n, None, n - 64, n) as job:  # warm-up
                job.add_variants(packed[:4096])
                job.counts()
            full_s, _ = timed(lambda: KingJob(ctx, n), False)
            res["runs"].append({"samples": n, "route": "full", "pairs": n * (n - 1) // 2, "device_s": full_s})
            print(json.dumps(res["runs"][-1]), flush=True)
            for f in args.fractions:
                r = max(1, int(round(f * n)))
                req = np.sort(rng.choice(n, size=r, replace=False))
                mask = np.zeros(n, dtype=bool)
                mask[req] = True
                order = np.concatenate([np.flatnonzero(~mask), np.flatnonzero(mask)]).astype(np.uint32)
                n0 = n - r
                pairs = (n * (n - 1) - n0 * (n0 - 1)) // 2
                dense_s, dense_rb = timed(lambda: MappedKingJob(ctx, n, order, n0, n), pairs * 20 <= 4 << 30)
                row = {"samples": n, "required": r, "route": "dense", "pairs": pairs, "device_s": dense_s, "readback_s": dense_rb,
                       "vs_full": round(full_s / dense_s, 2)}
                if pairs <= args.max_list_pairs:
                    jj = np.concatenate([np.full(j, j, dtype=np.uint32) for j in range(n0, n)])
                    ii = np.concatenate([np.arange(j, dtype=np.uint32) for j in range(n0, n)])
                    plist = np.stack([order[ii], order[jj]], axis=1)
                    list_s, list_rb = timed(lambda: KingPairJob(ctx, n, plist), True)
                    row.update(list_s=list_s, list_readback_s=list_rb, vs_list=round((list_s + list_rb) / (dense_s + dense_rb), 2))
                else:
                    row.update(list_s=None, list_note="pair list not run: %d pairs over --max-list-pairs" % pairs)
                res["runs"].append(row)
                print(json.dumps(row), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
