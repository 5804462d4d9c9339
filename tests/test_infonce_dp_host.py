"""CPU: data-parallel InfoNCE with global negatives (DESIGN.md section 7) -- the decomposition every rank runs, restated in
float64 on top of tests/infonce_oracle.py, exchanged with dib_b200.parallel over gloo, equals the one-process InfoNCE
loss and gradients; the loss object's ``negatives`` argument; the ctypes table of the three shard entry points against
include/dib_b200.h."""
import os
import re
import socket
from ctypes import c_int32, c_int64, c_uint32, c_uint64, c_void_p

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import dib_oracle as O
from tests import infonce_oracle as IO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def pair_similarity_grads(a, b, similarity, T):
    """S[i, j] = S(a_i, b_j) and its derivatives d S_ij / d a_i, d S_ij / d b_j ([p, q, d] each), the forms of
    IO.infonce_loss_and_grads."""
    S = O.get_scaled_similarity(a, b, similarity, T)
    diff = a[:, None, :] - b[None, :, :]
    if similarity == "cosine":
        na, nb = np.linalg.norm(a, axis=-1), np.linalg.norm(b, axis=-1)
        ah, bh = a / na[:, None], b / nb[:, None]
        c = ah @ bh.T
        ga = (bh[None, :, :] - c[:, :, None] * ah[:, None, :]) / na[:, None, None] / T
        gb = (ah[:, None, :] - c[:, :, None] * bh[None, :, :]) / nb[None, :, None] / T
        return S, ga, gb
    if similarity == "l2sq":
        ga = -2.0 * diff / T
    elif similarity == "l2":
        ga = -diff / (-S * T)[:, :, None] / T
    elif similarity == "l1":
        ga = -np.sign(diff) / T
    else:
        k = np.abs(diff).argmax(-1)
        ga = np.zeros_like(diff)
        ii, jj = np.meshgrid(np.arange(a.shape[0]), np.arange(b.shape[0]), indexing="ij")
        ga[ii, jj, k] = -np.sign(diff[ii, jj, k]) / T
    return S, ga, -ga


def rank_step(e1, e2, lo, hi, similarity, T):
    """One rank owning rows [lo, hi): the three phases and the exchanges of DESIGN.md section 7 in float64.  Returns the
    all-reduced loss sum and the all-gathered [d e1 || d e2] rows of the global batch."""
    from dib_b200 import parallel
    n, d = e1.shape
    own = np.arange(hi - lo)
    # phase 1: the own rows of e_all = (e1 || e2); exchange 1
    e_all = torch.zeros(n, 2 * d, dtype=torch.float64)
    e_all[lo:hi] = torch.from_numpy(np.concatenate([e1[lo:hi], e2[lo:hi]], 1))
    parallel.all_gather_rows_(e_all)
    E1, E2 = e_all[:, :d].numpy(), e_all[:, d:].numpy()
    # phase 2: r of the own e1 rows against all e2, c of the own e2 rows against all e1, s_ii; exchange 2
    S_row, ga_row, _ = pair_similarity_grads(E1[lo:hi], E2, similarity, T)
    S_col, _, gb_col = pair_similarity_grads(E1, E2[lo:hi], similarity, T)
    r_own, c_own = O._logsumexp(S_row, 1), O._logsumexp(S_col, 0)
    diag = S_row[own, lo + own]
    lse_all = torch.zeros(n, 2, dtype=torch.float64)
    lse_all[lo:hi] = torch.from_numpy(np.stack([r_own, c_own], 1))
    parallel.all_gather_rows_(lse_all)
    r_all, c_all = lse_all[:, 0].numpy(), lse_all[:, 1].numpy()
    # phase 3: d e1 of the own rows against all columns, d e2 of the own columns against all rows, weights / n_global
    W = (np.exp(S_row - r_own[:, None]) + np.exp(S_row - c_all[None, :])) / n
    W[own, lo + own] -= 2.0 / n
    d1 = np.einsum("ij,ijk->ik", W, ga_row)
    W2 = (np.exp(S_col - r_all[:, None]) + np.exp(S_col - c_own[None, :])) / n
    W2[lo + own, own] -= 2.0 / n
    d2 = np.einsum("ij,ijk->jk", W2, gb_col)
    # exchange 3: the stats are summed; the d e rows are gathered here only to compare them
    stats = torch.tensor([float((r_own + c_own - 2.0 * diag).sum()), float(hi - lo)], dtype=torch.float64)
    parallel.allreduce_sum_(stats)
    d_all = torch.zeros(n, 2 * d, dtype=torch.float64)
    d_all[lo:hi] = torch.from_numpy(np.concatenate([d1, d2], 1))
    parallel.all_gather_rows_(d_all)
    return stats.numpy(), d_all.numpy()


def data(n, d, seed):
    rng = np.random.default_rng(seed)
    e1 = rng.standard_normal((n, d))
    return e1, 0.6 * e1 + 0.8 * rng.standard_normal((n, d))


def _worker(rank, world, port, n, similarity, out_path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="2")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dib_b200 import parallel
        e1, e2 = data(n, 5, 0)                               # the same global batch on every rank
        lo, hi = parallel.shard_range(n, rank, world)
        assert hi - lo == n // world
        stats, d_all = rank_step(e1, e2, lo, hi, similarity, 0.5 if similarity == "cosine" else 1.0)
        if rank == 0:
            np.savez(out_path, stats=stats, d_all=d_all)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("similarity", O.SIMILARITY_TYPES)
def test_decomposition_over_gloo_is_the_one_process_infonce(tmp_path, world, similarity):
    n = 24
    out = str(tmp_path / "rank0.npz")
    mp.spawn(_worker, args=(world, _free_port(), n, similarity, out), nprocs=world, join=True)
    got = np.load(out)
    e1, e2 = data(n, 5, 0)
    loss, d1, d2 = IO.infonce_loss_and_grads(e1, e2, similarity, 0.5 if similarity == "cosine" else 1.0)
    assert got["stats"][1] == n
    assert abs(got["stats"][0] / n - loss) <= 1e-12 * max(1.0, abs(loss))
    np.testing.assert_allclose(got["d_all"][:, :5], d1, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got["d_all"][:, 5:], d2, rtol=0, atol=1e-12)


def test_all_gather_rows_is_a_no_op_in_one_process():
    from dib_b200 import parallel
    t = torch.arange(6.0).reshape(3, 2)
    assert parallel.all_gather_rows_(t) is t and torch.equal(t, torch.arange(6.0).reshape(3, 2))


def test_negatives_argument():
    from dib_b200 import losses
    assert losses.InfoNCE(6).negatives is None
    assert losses.InfoNCE(6, negatives="global").negatives == "global"
    for bad in ("local", "all", True):
        with pytest.raises(ValueError, match="negatives"):
            losses.InfoNCE(6, negatives=bad)


_CTYPES = {"dib_model*": c_void_p, "void*": c_void_p, "int64_t": c_int64, "int32_t": c_int32, "uint64_t": c_uint64,
           "uint32_t": c_uint32}


@pytest.mark.parametrize("name", ["dib_infonce_shard_forward", "dib_infonce_shard_lse", "dib_infonce_shard_backward"])
def test_shard_entry_points_ctypes_match_the_header(name):
    from dib_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dib_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    want = []
    for arg in m.group(1).split(","):
        toks = arg.replace("const ", "").split()
        typ = toks[0] + ("*" if "*" in arg else "")
        want.append(c_void_p if typ.endswith("*") else _CTYPES[typ])
    res, args = _lib.SIGNATURES[name]
    assert res is c_int32
    assert args == want, (name, args, want)
