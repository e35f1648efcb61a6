"""Operand traffic of the default KING kernel (`tensor_ts`, king_b1_kernel) on one GPU.

Times the kernel on a `--samples` x `--variants` random block with the library's CUDA events (as
`king_b1_rate.py --king` does) and states the operand bytes it pulls per second: each 128 x 64 pair tile reads
12 KB per 256 variants (8 KB of row words, 4 KB of column words of the sample-major copy), counted over the job's
tile list.  Set against the L2 bandwidth, this tells whether operand traffic or the tensor pipe
(`king_b1_rate.py --king`, `frac_of_b1_peak`) bounds the kernel.

    python tests/harness/king_b1_traffic.py [--reps 3] [--samples 16384] [--variants 65536] [--out DIR/king_b1_traffic.json]

The card name and power limit are read with nvidia-smi in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from king_b1_rate import card  # noqa: E402

KB1_TILE_COLS = 64
OPERAND_BYTES_PER_TILE_K256 = 8 * 128 * 8 + 8 * KB1_TILE_COLS * 8  # row words + column words of one k256 step


def king_tile_count(n):
    # the default KING tile list of rows [0, n) without the diagonal: row tile rt needs columns up to its last row - 1
    return sum(-(-(min(128 * (rt + 1), n) - 1) // KB1_TILE_COLS) for rt in range(-(-n // 128)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--samples", type=int, default=16384)
    ap.add_argument("--variants", type=int, default=65536)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np

    import plink_ng_b200 as p
    from plink_ng_b200.host import KING_ALGO_TENSOR_TS, KingJob, pack_genotypes

    n, m = args.samples, args.variants
    rng = np.random.default_rng(1)
    packed = pack_genotypes(rng.integers(0, 4, size=(m, n), dtype=np.uint8))
    tiles = king_tile_count(n)
    operand_bytes = tiles * OPERAND_BYTES_PER_TILE_K256 * (-(-m // 256))
    ms = []
    with p.GpuContext(0) as ctx:
        for _ in range(args.reps):
            with KingJob(ctx, n, 0, n, KING_ALGO_TENSOR_TS) as job:
                job.add_variants(packed)
                ms.append(job.last_kernel_ms())
    res = {"card": card(), "samples": n, "variants": m, "tiles": tiles, "operand_bytes": operand_bytes,
           "kernel_ms": [round(x, 3) for x in ms], "operand_tb_per_s": [round(operand_bytes / (x * 1e-3) / 1e12, 2) for x in ms]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
