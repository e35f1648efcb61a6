"""Tensor-pipe rates behind the binary (AND-POPC) KING kernel, on one GPU.

Runs the wgmma self-test (int8 and binary forms), then the chip-wide rate probes of `pl2gpu_int8_peak`:
int8 m64nNk32 (form 1) and b1 m64nNk256 AND-POPC (form 2) at N = 64 and 128, alternating, `--reps` times each.
For each N it reports c = (cycles of one b1 k256 wgmma) / (cycles of one int8 k32 wgmma) = 8 x int8 rate / b1 rate,
both rates counted as 2 M N K operations with K in elements (bits for b1).  With `--king` it also times the default
KING kernel (`tensor_ts`) on a `--samples` x `--variants` random block with CUDA events and states its rate as
bit AND-POPC operations (6 products of 2 n m^2 / 2) over the measured b1 peak.

    python tests/harness/king_b1_rate.py [--reps 3] [--king] [--out DIR/king_b1_rate.json]

The card name and power limit are read with nvidia-smi in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--king", action="store_true")
    ap.add_argument("--samples", type=int, default=16384)
    ap.add_argument("--variants", type=int, default=65536)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np

    import plink_ng_b200 as p
    from plink_ng_b200.host import KING_ALGO_TENSOR_TS, KingJob, pack_genotypes

    res = {"card": card()}
    with p.GpuContext(0) as ctx:
        ctx.selftest_umma(verbose=True)
        res["selftest"] = "ok"
        rates = {}
        for _ in range(args.reps):
            for n in (64, 128):
                for form, name in ((1, "int8"), (2, "b1")):
                    tops, _ = ctx.int8_peak(n, form, args.seconds)
                    rates.setdefault(f"{name}_n{n}", []).append(round(tops, 1))
        res["tops"] = rates
        res["c"] = {f"n{n}": [round(8 * i / b, 3) for i, b in zip(rates[f"int8_n{n}"], rates[f"b1_n{n}"])] for n in (64, 128)}
        if args.king:
            rng = np.random.default_rng(1)
            n, m = args.samples, args.variants
            geno = rng.integers(0, 4, size=(m, n), dtype=np.uint8)
            packed = pack_genotypes(geno)
            ms = []
            for _ in range(args.reps):
                with KingJob(ctx, n, 0, n, KING_ALGO_TENSOR_TS) as job:
                    job.add_variants(packed)
                    ms.append(job.last_kernel_ms())
            ops = 6 * 2.0 * m * n * (n + 1) / 2  # pairs incl. the diagonal; padding not counted
            b1_peak = max(rates["b1_n128"] + rates["b1_n64"])
            res["king"] = {"samples": n, "variants": m, "kernel_ms": [round(x, 3) for x in ms],
                           "b1_tops": [round(ops / (x * 1e-3) / 1e12, 1) for x in ms],
                           "frac_of_b1_peak": [round(ops / (x * 1e-3) / 1e12 / b1_peak, 3) for x in ms]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
