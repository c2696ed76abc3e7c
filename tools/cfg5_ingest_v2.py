"""The V2 reconcile cycle (BASELINE configs[4] for the token-based path): batch arrival -> V2 VariantDecisions, two ways
on the same seeded batches, alternated batch by batch:
  ingest_v2  the collector writes the six vectors into wva_ingest_v2's columns -> analyze (one graph launch) -> the host
             store step -> decide (one graph launch) -> decisions      (pipeline.ingest_v2_decisions)
  host       the collector's join on the host (tests/collector_v2_ref.collect, pod by pod) -> SaturationAnalyzerV2 with
             the history on the device -> CostAwareOptimizer -> Enforcer per model   (pipeline.optimize_v2)
Each path keeps its own capacity store and k2 history; the script asserts equal decisions and equal stores every batch
and prints one JSON line with p50 / p99 per path, the ingest_v2 path split into its parts (the device time of each graph
launch, the collector's writes, the host step), the card and its power limit.  Every model has `max_variants` variants.
Usage: cfg5_ingest_v2.py [models=10000] [batches=6] [max_variants=32]"""
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
from tests import collector_v2_ref as cv  # noqa: E402

M = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000
B = int(sys.argv[2]) if len(sys.argv) > 2 else 6
MV = int(sys.argv[3]) if len(sys.argv) > 3 else 32


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    fl = cv.fleet(M, MV, seed=M, exact=True)                       # every model MV variants, 0-4 pods each
    reg = cv.Registry(fl)
    batches = [cv.cycle(fl, 7000 + b) for b in range(B)]           # generated before any timing
    e = pkg.Engine(0)
    an_i, an_h = pkg.SaturationAnalyzerV2(e), pkg.SaturationAnalyzerV2(e, device_history=True)
    reg.seed_store(an_i.store); reg.seed_store(an_h.store)
    opt = pkg.CostAwareOptimizer(e)
    lat = {"ingest_v2": [], "host": []}
    dev = {"analyze_graph": [], "decide_graph": [], "host_step_and_decisions": [], "collector_write": []}
    n_dec = 0
    with pkg.K2History(e, *reg.k2_registry()) as h, pkg.IngestV2(e, reg.mvo, reg.vso, reg.var_acc, reg.var_slot, h) as ing:
        for b, (vec, state, mod) in enumerate(batches):
            runs = {}
            for path in (("ingest_v2", "host") if b % 2 == 0 else ("host", "ingest_v2")):
                t0 = time.perf_counter()
                if path == "ingest_v2":
                    reg.write(ing, pkg._abi, vec, state, mod, an_i.store)
                    t1 = time.perf_counter()
                    runs[path] = pkg.ingest_v2_decisions(ing, an_i, *reg.decisions_args())
                    t2 = time.perf_counter()
                    dev["analyze_graph"].append(ing.analyze_ms); dev["decide_graph"].append(ing.decide_ms)
                    dev["host_step_and_decisions"].append((t2 - t1) * 1e3 - ing.analyze_ms - ing.decide_ms)
                    dev["collector_write"].append((t1 - t0) * 1e3)
                else:
                    inputs, s2z, count, _ = reg.reference_inputs(vec, state, mod)
                    runs[path] = pkg.optimize_v2(an_h, opt, pkg.Enforcer(e, count), inputs, s2z)
                lat[path].append((time.perf_counter() - t0) * 1e3)
            assert runs["ingest_v2"] == runs["host"], "batch %d: the two paths decided differently" % b
            assert list(an_i.store.records.items()) == list(an_h.store.records.items()), "batch %d: stores differ" % b
            n_dec = len(runs["host"])
    an_h.close()
    e.close()
    warm = {k: v[1:] if len(v) > 2 else v for k, v in lat.items()}  # the first batch of each path builds its handles
    out = {"config": "cfg5_ingest_v2", "models": M, "variants": len(reg.var), "pods": len(reg.slot_of), "batches": B,
           "decisions_per_batch": n_dec, "decisions_equal": True, "card": card()}
    for k, v in warm.items():
        out[k + "_p50_ms"] = round(float(np.percentile(v, 50)), 2)
        out[k + "_p99_ms"] = round(float(np.percentile(v, 99)), 2)
    # where the ingest_v2 path's time goes: the two graphs (device time, CUDA events around each launch), the Python
    # collector writing the six vectors and the columns, and the host step + decision dicts around the launches
    out["ingest_v2_parts_p50_ms"] = {k: round(float(np.percentile(v[1:] if len(v) > 2 else v, 50)), 3) for k, v in dev.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
