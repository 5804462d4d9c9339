"""Generates tests/golden/ref_ctw.npz and ref_ctw_fresh.npz from the REFERENCE'S OWN native code: chaos/cppctw.cpp
compiled where it lies (oracle/Makefile -> oracle/_ref/libctw_ref.so; needs a checkout of the reference, REF=<dir>):
    make -C oracle REF=<reference checkout> && python tests/golden/make_ctw_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import ctw_oracle  # noqa: E402


def sequences():
    rng = np.random.default_rng(7)
    out = {"kat_1001": (np.array([1, 0, 0, 1]), 2),                     # chaos/setup.py:26-28 smoke call
           "zeros_1000": (np.zeros(1000, dtype=np.int64), 2),
           "alternating_1000": (np.arange(1000) % 2, 2),
           "single": (np.array([0]), 2)}
    lcg, v = [], 12345                                                   # SURVEY section 4: 20 000 LCG symbols, A = 4
    for _ in range(20000):
        v = (1103515245 * v + 12345) % (1 << 31)
        lcg.append((v >> 16) & 3)
    out["lcg_20000"] = (np.array(lcg), 4)
    x, sym = 0.3, []
    for _ in range(6000):                                                # a chaotic source (logistic map, r = 3.9)
        x = 3.9 * x * (1 - x)
        sym.append(int(x > 0.5))
    out["logistic_6000"] = (np.array(sym), 2)
    out["periodic_7x300"] = (np.tile([0, 1, 1, 2, 0, 2, 1], 300), 3)
    out["blocks_deep"] = (np.concatenate([np.zeros(700), np.ones(700), np.zeros(700)]).astype(np.int64), 2)   # depth > 512
    for n, A in ((17, 2), (300, 3), (2500, 5), (4000, 16)):
        out[f"random_{n}_{A}"] = (rng.integers(0, A, n), A)
    return out


def fresh_sequences():
    """Seeded random sequences with a long run (deep tails, depth > 512), and 300 short ones over small alphabets with runs
    and periodic pieces that exercise the lazy tail extension (tests/test_ctw.py)."""
    rng = np.random.default_rng(123)
    fresh = []
    for n, A in ((1, 3), (33, 2), (1000, 3), (6000, 4), (3000, 27)):
        seq = rng.integers(0, A, n)
        seq[n // 3: n // 3 + min(n // 4, 900)] = seq[0]
        fresh.append((seq, A))
    rng = np.random.default_rng(2024)
    small = []
    for trial in range(300):
        A = int(rng.integers(1, 6))
        n = int(rng.integers(1, 90))
        kind = trial % 3
        if kind == 0:
            seq = rng.integers(0, A, n)
        elif kind == 1:                                                       # runs
            seq = np.repeat(rng.integers(0, A, max(n // 7, 1)), 7)[:n]
        else:                                                                 # periodic with a defect
            seq = np.tile(rng.integers(0, A, int(rng.integers(1, 5))), n)[:n]
            seq[int(rng.integers(0, n))] = int(rng.integers(0, A))
        small.append((seq, A))
    return {"fresh": fresh, "small": small}


def main():
    assert ctw_oracle.reference_available(), "run `make -C oracle REF=<reference checkout>` first"
    rec = {}
    for name, (seq, A) in sequences().items():
        rec[name + "_seq"] = seq.astype(np.int8)
        rec[name + "_A"] = np.int32(A)
        rec[name + "_H"] = np.float64(ctw_oracle.reference_estimate_entropy(seq, A))
        print(f"{name:>20s}  A={A:<3d} n={len(seq):<6d} H={rec[name + '_H']!r}")
    np.savez_compressed(os.path.join(HERE, "ref_ctw.npz"), **rec)
    # sets of sequences: concatenated symbols, offsets, alphabet sizes, the reference's estimates
    rec = {}
    for name, cases in fresh_sequences().items():
        rec[name + "_seqs"] = np.concatenate([seq for seq, _ in cases]).astype(np.int8)
        rec[name + "_offsets"] = np.cumsum([0] + [len(seq) for seq, _ in cases]).astype(np.int64)
        rec[name + "_A"] = np.array([A for _, A in cases], dtype=np.int32)
        rec[name + "_H"] = np.array([ctw_oracle.reference_estimate_entropy(seq, A) for seq, A in cases], dtype=np.float64)
        print(f"{name:>20s}  {len(cases)} sequences, H[:3]={rec[name + '_H'][:3]!r}")
    np.savez_compressed(os.path.join(HERE, "ref_ctw_fresh.npz"), **rec)


if __name__ == "__main__":
    main()
