"""Per-cycle cost of a server set change on BASELINE configs[2] (100 000 models x 32 variants, N = 256, R = 256;
synth.baseline_config(3)), against a full reload of the same new system.

For the frontier-only grid and for full outputs, and for each cycle kind (0.1 %, 1 % and 10 % of the servers removed
and as many new ones added at random positions, the new ones with a neighbour's columns and a new load; and an SLO
edit on 1 % of the servers with the set unchanged): from a loaded, calculated and gridded system,
update_server_set + recalculate + grid_update, timed on the host around the three calls (each ends in a device
synchronise), then load_system + calculate + grid_run of the same new system on the same context, timed the same
way.  The first round checks that the two give bit-equal candidates and grids (the grid through a 64-bit sum and xor
of its words per field, perf_grid_update.digest).  A last, profiled set update per kind gives the re-index kernel's
time (torch.profiler, CUDA activities), and its achieved bytes/s: every byte it writes plus every kept byte it reads,
over that time, against the 3.35 TB/s of the H100 SXM data sheet.  Prints one JSON line with the card and its power
limit.

Usage: python tools/perf_server_set.py [--rounds 3] [--scale 1.0] [--R 256]
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

SRV = [k for k, (_, e) in pkg._abi.SYSTEM_ARRAYS.items() if e == "S"]
KINDS = (("churn", 0.001), ("churn", 0.01), ("churn", 0.1), ("slo", 0.01))
CAND_BYTES = sum(np.dtype(dt).itemsize for dt in pkg._abi.CAND_ARRAYS.values())   # per (server, accelerator)
LEVEL_BYTES = 1 + 4 * 4                                                              # ok + ttft, itl, rho, tput
HBM_PEAK = 3.35e12


def next_system(d, g, kind, f):
    """(new system, prev): `kind` "churn" removes round(f * S) servers and adds as many at random positions; "slo" edits
    the ITL SLO of f * S servers"""
    S = int(d["n_servers"])
    k = int(round(f * S))
    n = dict(d)
    if kind == "slo":
        for c in SRV:
            n[c] = d[c].copy()
        i = g.permutation(S)[:k]
        n["srv_slo_itl"][i] = (n["srv_slo_itl"][i] + np.float32(5.0)).astype(np.float32)
        return n, np.arange(S, dtype=np.int32)
    kept = np.sort(g.permutation(S)[k:])
    added = np.zeros(S, bool)
    added[g.choice(S, k, replace=False)] = True
    donors = g.integers(0, S, k)
    prev = np.full(S, -1, np.int32)
    prev[~added] = kept
    for c in SRV:
        col = np.empty(S, d[c].dtype)
        col[~added] = d[c][kept]
        col[added] = d[c][donors]
        n[c] = col
    n["srv_arrival"][added] = np.round(n["srv_arrival"][added] * np.float32(1.1) + np.float32(0.01), 2).astype(np.float32)
    return n, prev


def reindex_kernel_ms(e, prev, n):
    """one more set update under torch.profiler: the summed device time of the re-index kernel launches"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        e.update_server_set(prev, n)
        torch.cuda.synchronize()
    us = sum(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
             for ev in p.key_averages() if "reindex_rows_kernel" in ev.key)
    return us / 1e3


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
            for kind, f in KINDS:
                row = mode.setdefault(f"{kind} {f}", {"update_ms": [], "reload_ms": [], "resized": [], "regridded": []})
                for r in range(args.rounds + 1):                 # round 0 warms every launch shape up
                    e.load_system(base)
                    e.calculate()
                    e.grid_run(R, full=full)
                    n, prev = next_system(base, g, kind, f)
                    t0 = time.perf_counter()
                    e.update_server_set(prev, n)
                    rz, _ = e.recalculate()
                    rg = e.grid_update()
                    t1 = time.perf_counter()
                    if r == 1:
                        cand = e.candidates()
                        grid = digest(e, full, R, buf) if full else e.grid_fetch_frontier()
                    t2 = time.perf_counter()
                    e.load_system(n)
                    e.calculate()
                    e.grid_run(R, full=full)
                    t3 = time.perf_counter()
                    if r == 0:
                        continue
                    row["update_ms"].append(round((t1 - t0) * 1e3, 3))
                    row["reload_ms"].append(round((t3 - t2) * 1e3, 3))
                    row["resized"].append(rz)
                    row["regridded"].append(rg)
                    if r == 1:
                        c = e.candidates()
                        row["bit_equal"] = all(np.array_equal(cand[k].view(np.uint8), c[k].view(np.uint8))
                                               for k in c if k != "n_solves")
                        got = digest(e, full, R, buf) if full else e.grid_fetch_frontier()
                        row["bit_equal"] &= got == grid if full else np.array_equal(got, grid)
                if kind == "churn":                          # the re-index kernel, profiled in a run of its own
                    e.load_system(base)
                    e.calculate()
                    e.grid_run(R, full=full)
                    n, prev = next_system(base, g, kind, f)
                    ms = reindex_kernel_ms(e, prev, n)
                    kept = int((prev >= 0).sum())
                    per_row = A * (CAND_BYTES + 4) + (A * R * LEVEL_BYTES if full else 0)   # candidates, frontier, levels
                    moved = (S + kept) * per_row                 # written, plus read
                    row["reindex_kernel_ms"] = round(ms, 3)
                    row["reindex_bytes"] = moved
                    if ms > 0:
                        row["reindex_TBps"] = round(moved / (ms * 1e-3) / 1e12, 3)
                        row["reindex_share_of_3.35TBps"] = round(moved / (ms * 1e-3) / HBM_PEAK, 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
