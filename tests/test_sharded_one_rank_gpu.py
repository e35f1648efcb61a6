"""GPU: the sharded KING and GRM entry points on a one-rank NCCL communicator, so that a one-GPU machine runs the
path that `--gpus N` takes: the slice lands at row 0 of the staged block, is padded there, all-gathered in place
and counted.  Results must be bit-identical to the plain add of the same real rows."""
import numpy as np
import pytest
import torch

from plink_ng_b200 import GpuContext, Pl2Error, lib
from plink_ng_b200.capi import check
from plink_ng_b200.host import GrmJob, KingJob, comm_unique_id, pack_genotypes
from oracle import plink_oracle as orc

pytestmark = pytest.mark.gpu


def _random_geno(m, n, seed, miss=0.03):
    rng = np.random.default_rng(seed)
    freq = rng.uniform(0.02, 0.98, size=(m, 1))
    g = (rng.random((m, n)) < freq).astype(np.uint8) + (rng.random((m, n)) < freq).astype(np.uint8)
    g[rng.random((m, n)) < miss] = 3
    return g


@pytest.fixture
def one_rank_ctx():
    # a context of its own, so that the session context never carries a communicator (a second comm_init is refused)
    ctx = GpuContext(0)
    try:
        ctx.comm_init(0, 1, comm_unique_id())
    except Pl2Error as e:
        ctx.close()
        if "could not be loaded" in str(e):
            pytest.skip(str(e))
        raise
    try:
        yield ctx
    finally:
        ctx.comm_destroy()
        ctx.close()


# Real rows per slice; every slice is sent as SLICE rows, the missing ones topped up with all-missing rows (0xFF),
# as the host program tops up the last slice of a file.
SLICE = 700
REAL = [700, 431, 513]


@pytest.mark.parametrize("n", [150, 641], ids=lambda n: f"n{n}")
@pytest.mark.parametrize("src_is_device", [0, 2], ids=["host", "device"])
def test_king_sharded_matches_plain_add(one_rank_ctx, n, src_is_device):
    # 641 samples: the last 128-row tile holds one sample, the last 80-column tile one real column
    geno = _random_geno(sum(REAL), n, seed=n + src_is_device)
    packed = pack_genotypes(geno)
    blocks = np.full((len(REAL) * SLICE, packed.shape[1]), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    for k, real in enumerate(REAL):
        blocks[k * SLICE : k * SLICE + real] = packed[sum(REAL[:k]) : sum(REAL[: k + 1])]
    stride = blocks.strides[0]
    if src_is_device:
        dev = torch.from_numpy(blocks.view(np.uint8)).cuda()
        torch.cuda.synchronize()
        base = dev.data_ptr()
    else:
        base = blocks.ctypes.data
    with KingJob(one_rank_ctx, n) as job:
        for k in range(len(REAL)):
            job.add_variants_sharded(base + k * SLICE * stride, stride, SLICE, src_is_device)
        got = job.counts()
    with KingJob(one_rank_ctx, n) as job:
        job.add_variants(packed)
        plain = job.counts()
    assert np.array_equal(got, plain)
    assert np.array_equal(got, orc.king_counts(geno))


def test_grm_sharded_matches_plain_add(one_rank_ctx):
    n, slice_rows = 300, 1000
    batches = [_random_geno(m, n, seed=m) for m in (300, 777, 1000)]
    rng = np.random.default_rng(7)
    with GrmJob(one_rank_ctx, n) as job:
        for geno in batches:
            # rows past the batch are filler: random genotypes here, which must be ignored
            block = pack_genotypes(np.concatenate([geno, rng.integers(0, 4, size=(slice_rows - len(geno), n), dtype=np.uint8)]))
            check(lib.pl2gpu_grm_add_variants_sharded(job._h, block.ctypes.data, block.strides[0], slice_rows, len(geno), 0, None), "pl2gpu_grm_add_variants_sharded")
        g, obs = job.rows(with_obs=True)
    with GrmJob(one_rank_ctx, n) as job:
        for geno in batches:
            job.add_variants(pack_genotypes(geno))
        g_plain, obs_plain = job.rows(with_obs=True)
    assert np.array_equal(g, g_plain)
    assert np.array_equal(obs, obs_plain)
    _, want_obs = orc.grm(np.concatenate(batches))
    il = np.tril_indices(n)
    assert np.array_equal(obs[il], want_obs[il])
