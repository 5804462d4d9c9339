"""Float64 numpy oracle of the per-probe information map (nb-particle cell 8, :549-570; raw .ipynb line numbers), the
formula dib_mi_bounds_at_probes evaluates, in log space: equal to the notebook's linear-space densities wherever those do
not underflow, and finite where the notebook's upper bound becomes log(x / 0) = inf."""
import numpy as np

LOG_2PI = np.log(2.0 * np.pi)


def _lse(a, axis=-1):
    m = a.max(axis=axis, keepdims=True)
    return (m + np.log(np.exp(a - m).sum(axis=axis, keepdims=True))).squeeze(axis)


def mi_bounds_at_probes(probe_mu, probe_lv, data_mu, data_lv, eps, chunk=16):
    """probe_mu / probe_lv [M, E]; data_mu / data_lv: one [N_b, E] array per batch (a list, or a [B, N, E] array);
    eps [B, M, E].  Returns float64 [M, 2] = (mean_b lower_pb, mean_b upper_pb) in nats."""
    pm, pl = np.asarray(probe_mu, np.float64), np.asarray(probe_lv, np.float64)
    M, E = pm.shape
    c = -0.5 * E * LOG_2PI
    lower, upper = np.zeros(M), np.zeros(M)
    B = len(data_mu)
    for b in range(B):
        dm, dl = np.asarray(data_mu[b], np.float64), np.asarray(data_lv[b], np.float64)
        N = dm.shape[0]
        sig = np.exp(pl / 2.0)
        u = pm + sig * np.asarray(eps[b], np.float64)                                        # :554
        ls = -0.5 * (((u - pm) / sig) ** 2).sum(-1) - 0.5 * pl.sum(-1) + c                   # :557
        iv, cd = np.exp(-dl), -0.5 * dl.sum(-1) + c
        lse = np.empty(M)
        for a in range(0, M, chunk):
            d = u[a:a + chunk, None, :] - dm[None, :, :]
            lse[a:a + chunk] = _lse(-0.5 * (d * d * iv[None]).sum(-1) + cd[None])             # :563
        lower += ls - (np.logaddexp(ls, lse) - np.log(N + 1.0))                              # :566
        upper += ls - (lse - np.log(float(N)))                                               # :569
    return np.stack([lower / B, upper / B], axis=1)
