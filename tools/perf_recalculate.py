"""Per-cycle re-sizing cost against the share of servers whose load changed, on BASELINE configs[2] (100 000 models x
32 variants, N = 256; synth.baseline_config(3)).

One calculate, then for each changed share f: update_servers with the arrival rate of f * S servers moved by 0.01
req/min (the reference's two-decimal grid), recalculate, and a full calculate of the same system, alternated and
repeated.  Prints one JSON line: the card and its power limit, and per share the device time (calculate_ms) of every
recalculate and of every calculate next to it, the update's host wall time, and whether the recalculated candidates
were bit-equal to the calculated ones (checked in the first round; n_solves, the solve count of whichever sizer ran,
separately).

Usage: python tools/perf_recalculate.py [--rounds 3] [--scale 1.0]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("llm-d-workload-variant-autoscaler_b200")
CYCLE = tuple(pkg._abi.CYCLE_ARRAYS)
SHARES = (0.0, 0.001, 0.01, 0.1, 0.5, 1.0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except OSError:
        return "unknown"


def same(a, b, keys):
    return all(np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)) for k in keys)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    d = pkg.synth.baseline_config(3, scale=args.scale)
    S = int(d["n_servers"])
    cols = {k: d[k].copy() for k in CYCLE}
    g = np.random.default_rng(1)
    out = {"card": card(), "servers": S, "accelerators": int(d["n_acc"]), "rounds": args.rounds, "shares": {}}
    with pkg.Engine(0) as e:
        e.load_system(d)
        e.calculate()
        e.calculate()                                            # warm-up of every launch shape the calculate uses
        for f in SHARES:                                         # ... and of the recalculate at each share
            idx = g.permutation(S)[: int(round(f * S))]
            cols["srv_arrival"][idx] += np.float32(0.01)
            e.update_servers(*(cols[k] for k in CYCLE))
            e.recalculate()
        for r in range(args.rounds):
            for f in SHARES:
                row = out["shares"].setdefault(str(f), {"recalc_ms": [], "calc_ms": [], "update_wall_ms": [],
                                                        "resized": 0, "chain_solves": [], "sizer_kernel": []})
                idx = g.permutation(S)[: int(round(f * S))]
                cols["srv_arrival"][idx] += np.float32(0.01)
                t0 = time.perf_counter()
                e.update_servers(*(cols[k] for k in CYCLE))
                row["update_wall_ms"].append((time.perf_counter() - t0) * 1e3)
                row["resized"], _ = e.recalculate()
                t = e.timing()
                row["recalc_ms"].append(t["calculate_ms"])
                row["chain_solves"].append(t["chain_solves"])
                row["sizer_kernel"].append(t["sizer_kernel"])
                if r == 0:
                    rc = e.candidates()
                e.calculate()
                row["calc_ms"].append(e.timing()["calculate_ms"])
                if r == 0:                                       # n_solves: the solves of whichever sizer ran
                    c = e.candidates()
                    row["bit_equal"] = same(rc, c, [k for k in c if k != "n_solves"])
                    row["n_solves_equal"] = same(rc, c, ["n_solves"])
    for row in out["shares"].values():
        for k in ("recalc_ms", "calc_ms", "update_wall_ms"):
            row[k] = [round(x, 3) for x in row[k]]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
