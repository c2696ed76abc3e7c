"""Per-cycle cost of a table update on BASELINE configs[2] (100 000 models x 32 variants, N = 256, R = 256;
synth.baseline_config(3)), against a full wva_calculate + wva_grid_run of the same updated system.

For the frontier-only grid and for full outputs, and for each case (one accelerator's cost; alpha / beta / gamma of one
accelerator per model for 1 %, 10 % and 100 % of the models, as a tuner re-estimates them; every perf row): from a
loaded, calculated and gridded system, update_tables + recalculate + grid_update, then calculate + grid_run on the same
context, which then holds the same updated system.  Both are timed on the host around the calls (each ends in a device
synchronise) and by the device times the calls report (h2d_ms of the update, calculate_ms, grid_ms).  The first round
checks that the two give bit-equal candidates and grids (the grid through a 64-bit sum and xor of its words per field,
perf_grid_update.digest).  Prints one JSON line with the card and its power limit.

Usage: python tools/perf_table_update.py [--rounds 3] [--scale 1.0] [--R 256]
"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("llm-d-workload-variant-autoscaler_b200")
from perf_grid_update import card, digest  # noqa: E402

CASES = (("cost", 1.0), ("tuner", 0.01), ("tuner", 0.1), ("tuner", 1.0), ("all", 1.0))


def next_tables(d, g, kind, f):
    """a copy of d with its tables changed: "cost" one accelerator's cost, "tuner" alpha, beta and gamma of one
    accelerator per model on a share f of the models, "all" alpha of every perf row"""
    n = dict(d)
    A = int(d["n_acc"])
    if kind == "cost":
        n["acc_cost"] = d["acc_cost"].copy()
        n["acc_cost"][int(g.integers(0, A))] *= np.float32(1.05)
        return n
    if kind == "all":
        n["perf_alpha"] = (d["perf_alpha"] * np.float32(1.01)).astype(np.float32)
        return n
    M = d["perf_alpha"].size // A
    models = g.permutation(M)[: max(1, int(round(f * M)))]
    rows = models * A + g.integers(0, A, models.size)
    for k in ("perf_alpha", "perf_beta", "perf_gamma"):
        col = d[k].copy().reshape(-1)
        col[rows] = (col[rows] * np.float32(1.02)).astype(np.float32)
        n[k] = col.reshape(d[k].shape)
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--R", type=int, default=256)
    args = ap.parse_args()
    base = pkg.synth.baseline_config(3, scale=args.scale)
    S, A, R = int(base["n_servers"]), int(base["n_acc"]), args.R
    out = {"card": card(), "servers": S, "accelerators": A, "R": R, "rounds": args.rounds, "modes": {}}
    g = np.random.default_rng(1)
    buf = None
    with pkg.Engine(0) as e:
        for full in (False, True):
            if full and buf is None:
                buf = np.empty(S * A * R * 4 + 8, np.uint8)
            mode = out["modes"].setdefault("full" if full else "frontier", {})
            for kind, f in CASES:
                row = mode.setdefault(f"{kind} {f}", {"update_ms": [], "update_device_ms": [], "full_ms": [],
                                                      "full_device_ms": [], "marked_pairs": []})
                for r in range(args.rounds + 1):                 # round 0 warms every launch shape up
                    e.load_system(base)
                    e.calculate()
                    e.grid_run(R, full=full)
                    n = next_tables(base, g, kind, f)
                    t0 = time.perf_counter()
                    marked = e.update_tables(n)
                    dev = e.timing()["h2d_ms"]
                    e.recalculate()
                    dev += e.timing()["calculate_ms"]
                    e.grid_update()
                    dev += e.timing()["grid_ms"]
                    t1 = time.perf_counter()
                    if r == 1:
                        cand = e.candidates()
                        grid = digest(e, full, R, buf) if full else e.grid_fetch_frontier()
                    t2 = time.perf_counter()
                    e.calculate()
                    full_dev = e.timing()["calculate_ms"]
                    e.grid_run(R, full=full)
                    full_dev += e.timing()["grid_ms"]
                    t3 = time.perf_counter()
                    if r == 0:
                        continue
                    row["update_ms"].append(round((t1 - t0) * 1e3, 3))
                    row["update_device_ms"].append(round(dev, 3))
                    row["full_ms"].append(round((t3 - t2) * 1e3, 3))
                    row["full_device_ms"].append(round(full_dev, 3))
                    row["marked_pairs"].append(marked)
                    if r == 1:
                        c = e.candidates()
                        row["bit_equal"] = all(np.array_equal(cand[k].view(np.uint8), c[k].view(np.uint8))
                                               for k in c if k != "n_solves")
                        got = digest(e, full, R, buf) if full else e.grid_fetch_frontier()
                        row["bit_equal"] &= bool(got == grid if full else np.array_equal(got, grid))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
