"""Golden vectors for the per-probe information map by executing the NOTEBOOK'S OWN CODE on the numpy tf stand-in of
make_golden.py: nb-particle cell 8's inner probe lines (from ``embedding_dimension = tf.shape(mus_data)[-1]`` to
``upper_bounds_per.append(loo_per)``) are cut out of the cell text and exec'd verbatim, once per batch, with given probe /
data (mu, logvar) and queued eps.  The inputs keep every linear-space density far from underflow.

Needs the reference checkout (NB below); the tests only read its output:   python tests/golden/make_probe_golden.py
Writes tests/golden/ref_probe_information.npz (committed)."""
import json
import os
import sys
import textwrap

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G                                                # noqa: E402

NB = "/root/reference/complex_systems/InfoDecomp_Amorphous_plasticity_per_particle_measurements_and_set_transformer.ipynb"


def main():
    tf = G.install_tf_shim()
    cells = ["".join(c["source"]) for c in json.load(open(NB))["cells"] if c["cell_type"] == "code"]
    cell8 = next(c for c in cells if "upper_bounds_per.append(loo_per)" in c)
    a = cell8.index("embedding_dimension = tf.shape(mus_data)[-1]")
    a = cell8.rindex("\n", 0, a) + 1
    end = "upper_bounds_per.append(loo_per)"
    b = cell8.index(end) + len(end)
    src = textwrap.dedent(cell8[a:b])                                   # nb-particle cell 8, :549-570

    rng = np.random.default_rng(41)
    E, M, sizes = 4, 6, [5, 9, 3]
    probe_mu = 0.5 * rng.standard_normal((M, E))
    probe_lv = rng.uniform(-1.0, 0.0, (M, E))
    data_mu = 0.5 * rng.standard_normal((sum(sizes), E))
    data_lv = rng.uniform(-1.0, 0.0, (sum(sizes), E))
    eps = rng.standard_normal((len(sizes), M, E))
    off = np.concatenate([[0], np.cumsum(sizes)])
    lower, upper = [], []
    for bi in range(len(sizes)):
        G.EPS.q = [eps[bi]]
        ns = {"tf": tf, "np": np, "mus_data": data_mu[off[bi]:off[bi + 1]], "logvars_data": data_lv[off[bi]:off[bi + 1]],
              "mus_probes": probe_mu, "logvars_probes": probe_lv, "stddevs_probes": np.exp(probe_lv / 2.0),
              "probe_ind_start": 0, "probe_ind_end": M, "lower_bounds_per": [], "upper_bounds_per": []}
        exec(src, ns)
        assert not G.EPS.q
        lower.append(np.asarray(ns["lower_bounds_per"][0]))
        upper.append(np.asarray(ns["upper_bounds_per"][0]))
    out = dict(probe_mu=probe_mu, probe_lv=probe_lv, data_mu=data_mu, data_lv=data_lv, offsets=off, eps=eps,
               lower_per_batch=np.stack(lower), upper_per_batch=np.stack(upper))
    np.savez_compressed(os.path.join(HERE, "ref_probe_information.npz"), **out)
    print("probe golden: lower", out["lower_per_batch"].mean(0)[:3], "upper", out["upper_per_batch"].mean(0)[:3])


if __name__ == "__main__":
    main()
