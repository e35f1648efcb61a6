"""plink-ng_b200: H100-native (sm_90a) pairwise-genotype kernels behind PLINK 2.0's interfaces.

The product is the C-ABI shared library `libpl2gpu.so` (include/plink2_b200.h) and the `plink2_b200`
host program built from `plink_ng_b200/csrc`.  This Python package is only the ctypes binding used by
tests/ and bench.py; importing it never falls back to a CPU implementation.
"""
from .capi import lib, Pl2Error, last_error  # noqa: F401
from .host import (  # noqa: F401
    GpuContext,
    KingJob,
    pack_genotypes,
    unpack_genotypes,
    parallel_bounds,
    king_counts,
)
