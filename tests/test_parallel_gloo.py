"""CPU, world_size 2, gloo: the host-side data-parallel logic of the path -- contiguous row shards of each global
batch, local SUMS (gradients scaled by 1/B_global, statistics unscaled), one flat all-reduce(sum) of [grads || stats]
-- reproduces the single-process result.  The arithmetic inside each rank is done by the CPU oracle here (the CUDA
engine needs a GPU); the sharding / reduction code under test is dib_b200.parallel."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import dib_oracle as O
from tests.gpu_cases import _free_port


def _worker(rank, world, port, B, out_path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="2")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dib_b200 import parallel
    assert parallel.world_and_rank() == (world, rank)
    cfg = O.DIBConfig([1] * 3, [8], [8], 1, feature_embedding_dimension=4)
    rng = np.random.default_rng(0)                       # same data / params on every rank
    p = O.glorot_uniform_params(cfg, rng, dtype=np.float64)
    x, y = rng.standard_normal((B, 3)), rng.integers(0, 2, size=(B, 1)).astype(np.float64)
    eps = rng.standard_normal((B, 3, 4))                 # indexed by GLOBAL row
    lo, hi = parallel.shard_range(B, rank, world)
    g, fr = O.train_grads(cfg, p, x[lo:hi], y[lo:hi], eps[lo:hi], 0.3, O.LOSS_BCE_LOGITS, batch_for_mean=B)
    n = hi - lo
    stats = np.concatenate([fr.kl_per_feature * n, [fr.task_loss * n, fr.acc_sum, n]])
    flat = torch.from_numpy(np.concatenate([g, stats]))
    parallel.allreduce_sum_(flat)
    if rank == 0:
        np.save(out_path, flat.numpy())
    dist.destroy_process_group()


@pytest.mark.parametrize("B", [12, 13])
def test_two_rank_allreduce_matches_single_process(tmp_path, B):
    out = str(tmp_path / "flat.npy")
    mp.spawn(_worker, args=(2, _free_port(), B, out), nprocs=2, join=True)
    got = np.load(out)
    cfg = O.DIBConfig([1] * 3, [8], [8], 1, feature_embedding_dimension=4)
    rng = np.random.default_rng(0)
    p = O.glorot_uniform_params(cfg, rng, dtype=np.float64)
    x, y = rng.standard_normal((B, 3)), rng.integers(0, 2, size=(B, 1)).astype(np.float64)
    eps = rng.standard_normal((B, 3, 4))
    g, fr = O.train_grads(cfg, p, x, y, eps, 0.3, O.LOSS_BCE_LOGITS)
    want = np.concatenate([g, fr.kl_per_feature * B, [fr.task_loss * B, fr.acc_sum, B]])
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-13)
