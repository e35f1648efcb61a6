"""Operand-feed ceiling of the default KING kernel on one GPU: the bulk-copy read rate against bytes in flight.

`pl2gpu_bulk_read_rate` keeps a given number of bytes of 4 KB `cp.async.bulk` copies (global -> shared, onto
mbarriers, the instruction king_b1_kernel feeds itself with) in flight on every SM and reports TB/s.  This prints
that curve for a working set that stays in L2 (`--l2-mb`) and one that streams from HBM (`--hbm-gb`), then the
kernel's own operand rate (`king_b1_traffic.py`) beside it, with the kernel's SM cycles per tile-k256 step at the
card's maximum SM clock.

    python tests/harness/king_b1_feed.py [--inflight-kb 16,32,64,128,192] [--out DIR/king_b1_feed.json]

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
from king_b1_traffic import OPERAND_BYTES_PER_TILE_K256, king_tile_count  # noqa: E402


def measure(ctx, n, m, reps):
    """Kernel times of `reps` KING jobs on an n-sample x m-variant random block, their operand rates (as
    king_b1_traffic.py counts them) and the tile-k256 steps each SM runs."""
    import numpy as np
    import torch

    from plink_ng_b200.host import KING_ALGO_TENSOR_TS, KingJob, pack_genotypes

    packed = pack_genotypes(np.random.default_rng(1).integers(0, 4, size=(m, n), dtype=np.uint8))
    steps = king_tile_count(n) * -(-m // 256)
    ms = []
    for _ in range(reps):
        with KingJob(ctx, n, 0, n, KING_ALGO_TENSOR_TS) as job:
            job.add_variants(packed)
            ms.append(job.last_kernel_ms())
    return {"samples": n, "variants": m, "kernel_ms": [round(x, 3) for x in ms],
            "operand_tb_per_s": [round(steps * OPERAND_BYTES_PER_TILE_K256 / (x * 1e-3) / 1e12, 2) for x in ms],
            "tile_k256_steps_per_sm": steps / torch.cuda.get_device_properties(0).multi_processor_count}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inflight-kb", default="16,32,64,128,192")
    ap.add_argument("--l2-mb", type=int, default=16)
    ap.add_argument("--hbm-gb", type=int, default=4)
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=16384)
    ap.add_argument("--variants", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import plink_ng_b200 as p

    res = {"card": card()}
    inflight = [int(x) for x in args.inflight_kb.split(",")]
    with p.GpuContext(0) as ctx:
        for name, ws in (("l2", args.l2_mb << 20), ("hbm", args.hbm_gb << 30)):
            res[f"{name}_working_set_bytes"] = ws
            res[f"{name}_tb_per_s"] = {kb: round(ctx.bulk_read_rate(ws, kb << 10, args.seconds)[0], 3) for kb in inflight}
        king = measure(ctx, args.samples, args.variants, args.reps)
    try:
        mhz = float(res["card"].split(",")[2].split()[0])
        king["sm_cycles_per_tile_k256_at_max_clock"] = [round(ms * 1e-3 * mhz * 1e6 / king["tile_k256_steps_per_sm"]) for ms in king["kernel_ms"]]
    except (IndexError, ValueError):
        pass
    res["king_b1"] = king
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
