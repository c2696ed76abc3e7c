"""Where the replica grid's time goes on BASELINE configs[2] (or a scaled copy).

Builds the library of a source tree (default: this one) with -DWVA_GRID_PHASES into its own directory, runs the
materialised grid (R = 256) on the resident system and prints
  - the main pass's share of its warps' clock64() cycles: pair setup + head table, chain solves, and the rest (rates,
    admission, deferral, grid_store / eval_values, pair fetch);
  - the live lane-steps of the main pass (its states over the lock-step slots, 32 x the longest chain of a round), for
    a pair's first round and for its later rounds, and of the deferred pass;
  - the split of the grid's time between the main pass and grid_deferred_kernel (CUDA events around each).
The product library in the tree is neither used nor touched.

Usage: perf_grid_phases.py [--root TREE] [--out DIR] [--scale S] [--runs R] [--json FILE] [--lib SO]
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
NAMES = ["table", "chain", "total", "main_solves", "main_states", "main_states0",
         "main_ns", "deferred_ns", "slots0", "slots_rest", "slots_def", "rounds", "solves", "states", "certify_fallbacks"]


def build(tree: str, out: str) -> str:
    """copy the tree's csrc/ and include/ under `out` and build them there with the phase counters compiled in"""
    for sub in (os.path.join(PKG, "csrc"), "include"):
        dst = os.path.join(out, sub)
        shutil.rmtree(dst, ignore_errors=True)
        shutil.copytree(os.path.join(tree, sub), dst, ignore=shutil.ignore_patterns("*.so"))
    csrc = os.path.join(out, PKG, "csrc")
    subprocess.run(["sh", os.path.join(csrc, "build.sh"), "-DWVA_GRID_PHASES"], check=True, cwd=csrc,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return os.path.join(csrc, "libwva_b200.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT, help="source tree whose csrc/ is profiled")
    ap.add_argument("--out", help="build directory (default: a temporary one)")
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--R", type=int, default=256)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", help="also write the result here")
    ap.add_argument("--lib", help="a library already built with -DWVA_GRID_PHASES (nothing is built)")
    args = ap.parse_args()
    so = args.lib or build(os.path.abspath(args.root), args.out or tempfile.mkdtemp(prefix="grid_phases_"))

    sys.path.insert(0, ROOT)
    pkg = importlib.import_module(PKG)
    pkg.engine.lib_path = lambda: so
    d = pkg.synth.baseline_config(3, scale=args.scale)
    res = {"tree": os.path.abspath(args.root), "lib": so, "pairs": int(d["n_servers"] * d["n_acc"]), "R": args.R,
           "runs": []}
    with pkg.Engine(0) as e:
        e.lib.wva_grid_phases.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        e.load_system(d)
        e.grid_run(args.R, full=True)                                # warm-up
        print("warm-up grid: %.1f ms" % e.timing()["grid_ms"], flush=True)
        for _ in range(args.runs):
            e.lib.wva_grid_phases(e.ctx, None)
            e.grid_run(args.R, full=True)
            v = (C.c_uint64 * len(NAMES))()
            assert e.lib.wva_grid_phases(e.ctx, v) == 0
            r = dict(zip(NAMES, [int(x) for x in v]))
            r["grid_ms"] = e.timing()["grid_ms"]
            res["runs"].append(r)
    r = res["runs"][-1]
    tot = max(r["total"], 1)
    share = {"table": r["table"] / tot, "chain": r["chain"] / tot}
    share["rest"] = 1.0 - share["table"] - share["chain"]
    res["share"] = share
    slots = r["slots0"] + r["slots_rest"]
    live = {"main": r["main_states"] / max(slots, 1),
            "main_first_round": r["main_states0"] / max(r["slots0"], 1),
            "main_later_rounds": (r["main_states"] - r["main_states0"]) / max(r["slots_rest"], 1),
            "deferred": (r["states"] - r["main_states"]) / max(r["slots_def"], 1)}
    res["live_lane_steps"] = live
    res["main_ms"], res["deferred_ms"] = r["main_ns"] * 1e-6, r["deferred_ns"] * 1e-6
    print(f"replica grid, {res['pairs']} pairs x R = {args.R}, grid {', '.join('%.1f' % x['grid_ms'] for x in res['runs'])} ms")
    print(f"  main pass {res['main_ms']:.2f} ms, deferred pass {res['deferred_ms']:.2f} ms (last run, CUDA events)")
    print("  main pass, share of its warps' cycles:")
    print(f"    {'pair setup + head table':<44s} {100 * share['table']:6.2f} %")
    print(f"    {'chain solves':<44s} {100 * share['chain']:6.2f} %")
    print(f"    {'rest (rates, admission, deferral, stores)':<44s} {100 * share['rest']:6.2f} %")
    print(f"  main pass: {r['main_solves']} solves, {r['main_states']} states, {r['rounds']} rounds (both passes)")
    print(f"  live lane-steps: main {100 * live['main']:.1f} % (first rounds {100 * live['main_first_round']:.1f} %, "
          f"later rounds {100 * live['main_later_rounds']:.1f} %), deferred {100 * live['deferred']:.1f} %")
    print(f"  all passes: {r['solves']} solves, {r['states']} states, not certified (E12) {r['certify_fallbacks']}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
