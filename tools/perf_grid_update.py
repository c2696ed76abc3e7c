"""Per-cycle grid update cost against the share of servers whose load changed, on BASELINE configs[2] (100 000 models x
32 variants, N = 256, R = 256; synth.baseline_config(3)).

For full outputs and for the frontier alone: one grid_run, then for each changed share f: update_servers with the
arrival rate of f * S servers moved by 0.01 req/min (the reference's two-decimal grid), grid_update, and a full
grid_run of the same system, alternated and repeated.  Prints one JSON line: the card and its power limit, and per
mode and share the device time (grid_ms) of every grid_update and of every grid_run next to it, and whether the
updated grid was bit-equal to the one the grid_run gave (checked in the first round, field by field through a 64-bit
sum and xor of its words).

Usage: python tools/perf_grid_update.py [--rounds 3] [--scale 1.0] [--R 256]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("llm-d-workload-variant-autoscaler_b200")
CYCLE = tuple(pkg._abi.CYCLE_ARRAYS)
SHARES = (0.0, 0.001, 0.01, 0.1, 0.5, 1.0)
FIELDS = (("ok", 1), ("ttft", 4), ("itl", 4), ("rho", 4), ("tput", 4))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except OSError:
        return "unknown"


def digest(e, full, R, buf):
    """the resident grid, one field at a time through `buf`: (field, 64-bit sum, xor) of its words"""
    n_pairs = (e.hi - e.lo) * e.A
    out = []
    for k, width in (("frontier", 4),) + (FIELDS if full else ()):
        n = n_pairs * (1 if k == "frontier" else R) * width
        ptrs = [None] * 6
        ptrs[5 if k == "frontier" else [f for f, _ in FIELDS].index(k)] = buf.ctypes.data
        e._check(e.lib.wva_grid_fetch(e.ctx, *ptrs), "wva_grid_fetch")
        n8 = (n + 7) // 8 * 8
        buf[n:n8] = 0
        words = buf[:n8].view(np.uint64)
        out.append((k, int(words.sum(dtype=np.uint64)), int(np.bitwise_xor.reduce(words))))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--R", type=int, default=256)
    args = ap.parse_args()
    R = args.R
    d = pkg.synth.baseline_config(3, scale=args.scale)
    S, A = int(d["n_servers"]), int(d["n_acc"])
    out = {"card": card(), "servers": S, "accelerators": A, "R": R, "rounds": args.rounds, "modes": {}}
    buf = np.zeros(S * A * R * 4 + 8, np.uint8)               # the largest field, zero-padded to whole words
    g = np.random.default_rng(1)
    with pkg.Engine(0) as e:
        e.load_system(d)
        cols = {k: d[k].copy() for k in CYCLE}
        for full in (True, False):
            mode = out["modes"].setdefault("full" if full else "frontier", {})
            e.grid_run(R, full=full)
            e.grid_run(R, full=full)                             # warm-up of every launch shape the run uses
            for f in SHARES:                                     # ... and of the update at each share
                idx = g.permutation(S)[: int(round(f * S))]
                cols["srv_arrival"][idx] += np.float32(0.01)
                e.update_servers(*(cols[k] for k in CYCLE))
                e.grid_update()
            for r in range(args.rounds):
                for f in SHARES:
                    row = mode.setdefault(str(f), {"update_ms": [], "run_ms": [], "regridded": 0, "chain_solves": []})
                    idx = g.permutation(S)[: int(round(f * S))]
                    cols["srv_arrival"][idx] += np.float32(0.01)
                    e.update_servers(*(cols[k] for k in CYCLE))
                    row["regridded"] = e.grid_update()
                    t = e.timing()
                    row["update_ms"].append(round(t["grid_ms"], 3))
                    row["chain_solves"].append(t["chain_solves"])
                    if r == 0:
                        upd = digest(e, full, R, buf)
                    e.grid_run(R, full=full)
                    row["run_ms"].append(round(e.timing()["grid_ms"], 3))
                    if r == 0:
                        row["bit_equal"] = upd == digest(e, full, R, buf)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
