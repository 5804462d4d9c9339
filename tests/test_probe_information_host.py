"""Host tests of the per-probe information map: the float64 oracle against the notebook-line golden and closed forms, and the set-draw row / offset
arithmetic of utils.set_batch_rows for fixed and ragged sets."""
import numpy as np
import torch

from tests import probe_information_oracle as PO


def test_oracle_matches_the_notebook_golden():
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_probe_information.npz"))
    off = g["offsets"]
    dm = [g["data_mu"][off[b]:off[b + 1]] for b in range(len(off) - 1)]
    dl = [g["data_lv"][off[b]:off[b + 1]] for b in range(len(off) - 1)]
    out = PO.mi_bounds_at_probes(g["probe_mu"], g["probe_lv"], dm, dl, g["eps"])
    np.testing.assert_allclose(out[:, 0], g["lower_per_batch"].mean(0), rtol=0, atol=1e-12)
    np.testing.assert_allclose(out[:, 1], g["upper_per_batch"].mean(0), rtol=0, atol=1e-12)


def _probe(E, rng):
    return rng.standard_normal((1, E)), rng.uniform(-1.0, 0.5, (1, E))


def test_identical_rows_give_zero_information():
    rng = np.random.default_rng(0)
    E, N, B = 6, 9, 3
    pm, pl = _probe(E, rng)
    dm, dl = [np.repeat(pm, N, 0)] * B, [np.repeat(pl, N, 0)] * B
    out = PO.mi_bounds_at_probes(pm, pl, dm, dl, rng.standard_normal((B, 1, E)))
    np.testing.assert_allclose(out, 0.0, atol=1e-12)


def test_k_identical_rows_and_far_rows_give_the_counting_closed_form():
    rng = np.random.default_rng(1)
    E, N, k, B = 4, 12, 3, 2
    pm, pl = _probe(E, rng)
    sig = np.exp(pl / 2)
    far = pm + 1e3 * sig.max() * (1 + np.arange(N - k))[:, None]                 # >= 10^3 sigma away
    dm = [np.concatenate([np.repeat(pm, k, 0), far])] * B
    dl = [np.repeat(pl, N, 0)] * B
    out = PO.mi_bounds_at_probes(pm, pl, dm, dl, 0.3 * rng.standard_normal((B, 1, E)))
    np.testing.assert_allclose(out[0], [np.log((N + 1) / (k + 1)), np.log(N / k)], atol=1e-12)


def test_all_far_rows_give_log_n_plus_one_and_a_finite_upper_bound():
    # the notebook's linear-space upper bound is log(p_own / 0) = inf here; the log-space form stays finite (and large)
    rng = np.random.default_rng(2)
    E, N = 3, 7
    pm, pl = _probe(E, rng)
    dm = [pm + 1e3 * (1 + np.arange(N))[:, None]]
    dl = [np.repeat(pl, N, 0)]
    out = PO.mi_bounds_at_probes(pm, pl, dm, dl, 0.1 * rng.standard_normal((1, 1, E)))
    np.testing.assert_allclose(out[0, 0], np.log(N + 1), atol=1e-12)
    assert np.isfinite(out[0, 1]) and out[0, 1] > 1e5


def test_ragged_batches_are_independent_problems():
    rng = np.random.default_rng(3)
    E, M = 5, 4
    pm, pl = rng.standard_normal((M, E)), rng.uniform(-1, 0, (M, E))
    sizes = [1, 6, 3]
    dm = [rng.standard_normal((n, E)) for n in sizes]
    dl = [rng.uniform(-1, 0, (n, E)) for n in sizes]
    eps = rng.standard_normal((3, M, E))
    both = PO.mi_bounds_at_probes(pm, pl, dm, dl, eps)
    each = [PO.mi_bounds_at_probes(pm, pl, dm[b:b + 1], dl[b:b + 1], eps[b:b + 1]) for b in range(3)]
    np.testing.assert_allclose(both, np.mean(each, axis=0), atol=1e-12)
    # one data row: the lower bound is log 2 - log(1 + p_j / p_own) and the upper log p_own - log p_j
    one = each[0]
    assert np.all(one[:, 0] <= np.log(2.0) + 1e-12)


def test_set_batch_rows_fixed_sets():
    from dib_b200 import utils
    idx = torch.tensor([[2, 0], [1, 1]])
    rows, off = utils.set_batch_rows(idx, None, 3)
    assert rows.tolist() == [6, 7, 8, 0, 1, 2, 3, 4, 5, 3, 4, 5]
    assert off.tolist() == [0, 6, 12]


def test_set_batch_rows_ragged_sets_skip_padding():
    from dib_b200 import utils
    idx = torch.tensor([[2, 0, 2], [1, 3, 0]])
    sizes = torch.tensor([1, 3, 2, 4])
    rows, off = utils.set_batch_rows(idx, sizes, 4)
    assert rows.tolist() == [8, 9, 0, 8, 9] + [4, 5, 6, 12, 13, 14, 15, 0]
    assert off.tolist() == [0, 5, 13]
