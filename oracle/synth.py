"""Seeded synthetic PLINK 1 filesets for the at-scale parity tests (tests/test_scale_gpu.py).

Genotypes follow a simple linkage model so that LD pruning has work to do: variant k copies the genotypes of
variant k - 1 and redraws a fraction `redraw` of the samples under Hardy-Weinberg at its own ALT frequency
(~U(0.05, 0.5)); `miss` of all calls are then set missing.  The bytes depend only on the arguments (numpy's PCG64
stream), so the digests of the reference's outputs stored under tests/golden/ stay valid.
"""
import numpy as np

# dosage (ALT count) 0/1/2, missing = 3 -> .bed code (00 hom A1 = ALT, 01 missing, 10 het, 11 hom A2 = REF)
_BED_CODE = np.array([3, 2, 0, 1], dtype=np.uint8)


def synth_dosages(n, m, seed, miss=0.01, redraw=0.5):
    """uint8 [m, n]: ALT dosage 0/1/2 or 3 = missing."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(0.05, 0.5, m)
    out = np.empty((m, n), dtype=np.uint8)
    cur = rng.binomial(2, p[0], n).astype(np.uint8)
    for k in range(m):
        if k:
            mask = rng.random(n) < redraw
            cur = cur.copy()
            cur[mask] = rng.binomial(2, p[k], int(mask.sum()))
        out[k] = cur
    out[rng.random((m, n)) < miss] = 3
    return out


def write_bed(prefix, n, m, seed, miss=0.01, redraw=0.5):
    """prefix.bed/.bim/.fam with n samples and m variants on chromosome 1 (variant k at bp k + 1)."""
    d = synth_dosages(n, m, seed, miss, redraw)
    codes = _BED_CODE[d]
    pad = (-n) % 4
    if pad:
        codes = np.concatenate([codes, np.zeros((m, pad), dtype=np.uint8)], axis=1)
    q = codes.reshape(m, -1, 4)
    packed = q[:, :, 0] | (q[:, :, 1] << 2) | (q[:, :, 2] << 4) | (q[:, :, 3] << 6)
    with open(prefix + ".bed", "wb") as f:
        f.write(bytes([0x6C, 0x1B, 0x01]))
        packed.astype(np.uint8).tofile(f)
    with open(prefix + ".bim", "w") as f:
        f.write("".join(f"1\tsnp{k}\t0\t{k + 1}\tA\tG\n" for k in range(m)))
    with open(prefix + ".fam", "w") as f:
        f.write("".join(f"fam{k}\tid{k}\t0\t0\t0\t-9\n" for k in range(n)))
