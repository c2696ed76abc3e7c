"""Where the pool sizer's time goes on BASELINE configs[2] (or a scaled copy).

Builds the library of a source tree (default: this one) with -DWVA_POOL_PHASES into its own directory, runs
System.Calculate on the pool sizer and prints each phase's share of the warps' clock64() cycles, and the live
lane-steps of fast and exact batches.  The fast batches are split further into the model load (pool_load_model), the
first tile wait of each head pass, the head chunks (the later tile waits included) and fast_solve_finish, and the head
chunks' cycles are given per warp-state (one state index of a batch: 32 lane-steps, live or not) and per live lane-state.
The product library in the tree is neither used nor touched.

Usage: perf_pool_phases.py [--root TREE] [--out DIR] [--scale S] [--runs R] [--json FILE]
"""
import argparse
import ctypes as C
import importlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "llm-d-workload-variant-autoscaler_b200"
NAMES = ["lock", "new_pairs", "fast", "exact", "state", "total", "fast_batches", "fast_states", "fast_slots",
         "exact_batches", "exact_states", "exact_slots", "fast_partial", "exact_partial", "rows", "iters",
         "model", "fast_wait0", "fast_chunks", "fast_finish"]
PHASES = {"lock": "critical section", "new_pairs": "new-pair setup + BuildModel",
          "fast": "model load + fast head + finish", "exact": "exact solves",
          "state": "state load + sizer_on_solve + store"}
FAST_PARTS = {"model": "model load", "fast_wait0": "first tile wait", "fast_chunks": "head chunks",
              "fast_finish": "fast_solve_finish"}


def build(tree: str, out: str) -> str:
    """copy the tree's csrc/ and include/ under `out` and build them there with the phase counters compiled in"""
    for sub in (os.path.join(PKG, "csrc"), "include"):
        dst = os.path.join(out, sub)
        shutil.rmtree(dst, ignore_errors=True)
        shutil.copytree(os.path.join(tree, sub), dst, ignore=shutil.ignore_patterns("*.so"))
    csrc = os.path.join(out, PKG, "csrc")
    subprocess.run(["sh", os.path.join(csrc, "build.sh"), "-DWVA_POOL_PHASES"], check=True, cwd=csrc,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return os.path.join(csrc, "libwva_b200.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT, help="source tree whose csrc/ is profiled")
    ap.add_argument("--out", help="build directory (default: a temporary one)")
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", help="also write the result here")
    ap.add_argument("--lib", help="a library already built with -DWVA_POOL_PHASES (nothing is built)")
    args = ap.parse_args()
    so = args.lib or build(os.path.abspath(args.root), args.out or tempfile.mkdtemp(prefix="pool_phases_"))

    sys.path.insert(0, ROOT)
    pkg = importlib.import_module(PKG)
    pkg.engine.lib_path = lambda: so
    d = pkg.synth.baseline_config(3, scale=args.scale)
    res = {"tree": os.path.abspath(args.root), "lib": so, "pairs": int(d["n_servers"] * d["n_acc"]), "runs": []}
    with pkg.Engine(0) as e:
        e.lib.wva_pool_phases.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        e.set_option(1, 6)
        e.load_system(d)
        e.calculate()                                  # warm-up
        print("warm-up calculate: %.1f ms" % e.timing()["calculate_ms"], flush=True)
        for _ in range(args.runs):
            e.lib.wva_pool_phases(e.ctx, None)
            e.calculate()
            v = (C.c_uint64 * len(NAMES))()
            assert e.lib.wva_pool_phases(e.ctx, v) == 0
            t = e.timing()
            r = dict(zip(NAMES, [int(x) for x in v]))
            r.update(calculate_ms=t["calculate_ms"], chain_solves=t["chain_solves"], chain_states=t["chain_states"],
                     certify_fallbacks=t["certify_fallbacks"])
            res["runs"].append(r)
        e.set_option(1, 0)
    r = res["runs"][-1]
    tot = r["total"]
    share = {k: r[k] / tot for k in PHASES}
    share["idle"] = 1.0 - sum(share.values())
    res["share"] = share
    print(f"pool sizer phases, {res['pairs']} pairs, calculate {', '.join('%.1f' % x['calculate_ms'] for x in res['runs'])} ms")
    for k, txt in PHASES.items():
        print(f"  {txt:<40s} {100 * share[k]:6.2f} %")
    print(f"  {'idle (no request to take)':<40s} {100 * share['idle']:6.2f} %")
    parts = {k: r[k] / tot for k in FAST_PARTS}
    parts["fast_other"] = share["fast"] - sum(parts.values())
    res["fast_parts"] = parts
    print("  of which, fast batches:")
    for k, txt in FAST_PARTS.items():
        print(f"    {txt:<38s} {100 * parts[k]:6.2f} %")
    print(f"    {'rest (call, batch bookkeeping)':<38s} {100 * parts['fast_other']:6.2f} %")
    warp_states = r["fast_slots"] / 32
    res["chunk_cycles_per_warp_state"] = r["fast_chunks"] / max(warp_states, 1)
    res["chunk_cycles_per_live_lane_state"] = r["fast_chunks"] / max(r["fast_states"], 1)
    print(f"  head chunks: {res['chunk_cycles_per_warp_state']:.1f} cycles per warp-state "
          f"({warp_states:.3g} warp-states), {res['chunk_cycles_per_live_lane_state']:.2f} per live lane-state; "
          f"first tile wait {r['fast_wait0'] / max(r['fast_batches'], 1):.0f} cycles per batch")
    for kind in ("fast", "exact"):
        b, st, sl = r[f"{kind}_batches"], r[f"{kind}_states"], r[f"{kind}_slots"]
        print(f"  {kind} batches {b} ({r[kind + '_partial']} with < 32 requests): live lane-steps {st} of {sl} "
              f"({100 * st / max(sl, 1):.1f} %)")
    print(f"  rows built {r['rows']}, warp iterations {r['iters']}, solves {r['chain_solves']}, "
          f"not certified {r['certify_fallbacks']}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
