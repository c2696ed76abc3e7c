"""BASELINE configs[4]: streaming reconcile — 10 k-model Prometheus-shaped metric batches, batch arrival -> decisions,
INCLUDING the SoA packing (the collector's columnar writer), through wva_ingest_* (one CUDA graph per batch) + the
GPU-count limiter.  The `final_decisions` leg times batch arrival -> the cycle's final decisions (enforcer, decisions,
limiter) two ways on the same batches, alternated: the decision-mode graph (wva_ingest_create_decisions) and the plain
graph + enforcer / decisions on the host + wva_limit; it asserts both give the same decisions.
Usage: cfg5_ingest.py [models=10000] [batches=60]"""
import importlib, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("llm-d-workload-variant-autoscaler_b200")
M = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000
B = int(sys.argv[2]) if len(sys.argv) > 2 else 60


def measure(e, M, B, shuffled):
    # deployment: every model 32 variants, 1..8 pods each (the synthetic generator of config 4/5); registry = all pods
    d0 = pkg.synth.saturation_batch(M, 32, stream=500)
    V = d0["n_variants"]
    vso = d0["variant_replica_off"].astype(np.int32)           # every pod of the deployment has a slot
    S = int(vso[-1])
    ing = pkg.Ingest(e, d0["model_variant_off"], vso)
    acc_type, gpr = (np.arange(V) % 8).astype(np.int32), np.ones(V, np.int32)
    lat, parts = [], []
    g = np.random.default_rng(5)
    for b in range(B):
        d = pkg.synth.saturation_batch(M, 32, stream=500)       # same deployment (same seed -> same pods) ...
        kvv = np.random.default_rng(1000 + b).beta(2.0, 3.0, S)  # ... fresh metric values every cycle
        qv = np.random.default_rng(2000 + b).poisson(1.5, S).astype(np.float64)
        # two Prometheus vectors keyed by pod: (slot, value) pairs in response order; 2 % of the pods miss a cycle
        rep = np.flatnonzero(g.random(S) > 0.02).astype(np.int32)
        order = g.permutation(rep.size) if shuffled else np.arange(rep.size)
        slots = rep[order]
        kvs, qs = kvv[slots], qv[slots]
        limit = np.full(8, int(d["var_current"].sum() // 8 + 500), np.int32)
        t0 = time.perf_counter()
        ing.begin()
        ing.write(pkg._abi.VEC_KV_CACHE_USAGE, slots, kvs)
        ing.write(pkg._abi.VEC_QUEUE_LENGTH, slots, qs)
        ing.cols["var_cost"][:] = d["var_cost"]; ing.cols["var_current"][:] = d["var_current"]
        ing.cols["var_desired"][:] = d["var_desired"]; ing.cols["var_pending"][:] = d["var_pending"]
        for k in ("cfg_kv_threshold", "cfg_queue_threshold", "cfg_kv_trigger", "cfg_queue_trigger"):
            ing.cols[k][:] = d[k]
        t1 = time.perf_counter()
        r = ing.commit()
        t2 = time.perf_counter()
        gms = e.timing()["saturation_ms"]
        e.limit({"n_types": 8, "acc_type": acc_type, "current": d["var_current"], "target": np.maximum(r["var_target"], 0),
                 "gpus_per_replica": gpr, "spare": r["var_avg_spare_kv"], "cost": d["var_cost"], "type_limit": limit})
        t3 = time.perf_counter()
        lat.append((t3 - t0) * 1e3); parts.append(((t1 - t0) * 1e3, (t2 - t1) * 1e3, gms, (t3 - t2) * 1e3))
    ing.close()
    lat = np.array(lat[5:]); parts = np.array(parts[5:])
    return {"p50_ms": float(np.percentile(lat, 50)), "p99_ms": float(np.percentile(lat, 99)),
            "packing_ms_p50": float(np.percentile(parts[:, 0], 50)), "graph_wall_ms_p50": float(np.percentile(parts[:, 1], 50)),
            "graph_device_ms_p50": float(np.percentile(parts[:, 2], 50)), "limiter_ms_p50": float(np.percentile(parts[:, 3], 50)),
            "pods": S, "variants": int(V)}


def measure_decisions(e, M, B, T=8):
    """batch arrival -> final decisions, decision-mode graph vs plain graph + host + wva_limit, alternated per batch"""
    d0 = pkg.synth.saturation_batch(M, 32, stream=500)
    V, mvo = d0["n_variants"], d0["model_variant_off"].astype(np.int32)
    vso = d0["variant_replica_off"].astype(np.int32)
    S = int(vso[-1])
    model_of = np.repeat(np.arange(M), np.diff(mvo))
    new, old = pkg.Ingest(e, mvo, vso, n_types=T), pkg.Ingest(e, mvo, vso)
    g = np.random.default_rng(7)
    acc_type = np.where(g.random(V) < 0.05, -1, np.arange(V) % T).astype(np.int32)
    gpr = np.array([0, 1, 1, 2, 4])[g.integers(0, 5, V)].astype(np.int32)
    lat = {"graph": [], "graph_host_limit": []}
    decided = []

    def fill(ing, d, slots, kvs, qs, dc):
        ing.begin()
        ing.write(pkg._abi.VEC_KV_CACHE_USAGE, slots, kvs)
        ing.write(pkg._abi.VEC_QUEUE_LENGTH, slots, qs)
        for k in ("var_cost", "var_current", "var_desired", "var_pending", "cfg_kv_threshold", "cfg_queue_threshold",
                  "cfg_kv_trigger", "cfg_queue_trigger"):
            ing.cols[k][:] = d[k]
        if ing.dcols is not None:
            for k, v in dc.items():
                ing.dcols[k][:] = v

    def run_new(d, slots, kvs, qs, dc):
        fill(new, d, slots, kvs, qs, dc)
        new.commit()
        r = new.dres
        return {k: r[k].copy() for k in ("has_decision", "original_target", "target", "gpus_allocated", "was_limited", "action")}

    def run_old(d, slots, kvs, qs, dc):
        fill(old, d, slots, kvs, qs, dc)
        r = old.commit()
        va = r["var_replica_count"] > 0
        rep = np.bincount(model_of, weights=r["var_replica_count"], minlength=M) > 0
        tgt, _ = e.enforce(dict(model_variant_off=mvo, mod_scale_to_zero_enabled=dc["mod_scale_to_zero_enabled"],
                                mod_request_count=dc["mod_request_count"], mod_request_error=dc["mod_request_error"],
                                var_cost=d["var_cost"], var_has_cost=va.astype(np.uint8), var_target=r["var_target"]))
        has = rep[model_of] & (tgt >= 0)
        idx = np.flatnonzero(has)
        cur = d["var_current"]
        out = {"has_decision": has.astype(np.uint8), "original_target": np.where(has, tgt, -1).astype(np.int32),
               "target": np.where(has, tgt, -1).astype(np.int32), "gpus_allocated": np.zeros(V, np.int32),
               "was_limited": np.zeros(V, np.uint8), "action": np.where(has, np.sign(tgt - cur), 0).astype(np.int8)}
        if dc["enable_limiter"][0] and idx.size:
            lo = e.limit({"n_types": T, "acc_type": np.where(va, dc["var_accelerator_type"], -1)[idx], "current": cur[idx],
                          "target": tgt[idx], "gpus_per_replica": np.maximum(dc["var_gpus_per_replica"], 1)[idx],
                          "spare": np.where(va, r["var_avg_spare_kv"], 0.0)[idx], "cost": np.where(va, d["var_cost"], 0.0)[idx],
                          "type_limit": dc["type_limit"]})
            out["target"][idx], out["gpus_allocated"][idx], out["was_limited"][idx] = lo["target"], lo["gpus_allocated"], lo["was_limited"]
        return out

    for b in range(B):
        d = pkg.synth.saturation_batch(M, 32, stream=500)
        kvv = np.random.default_rng(1000 + b).beta(2.0, 3.0, S)
        qv = np.random.default_rng(2000 + b).poisson(1.5, S).astype(np.float64)
        slots = np.flatnonzero(g.random(S) > 0.02).astype(np.int32)
        kvs, qs = kvv[slots], qv[slots]
        used = np.bincount(acc_type.clip(0), weights=d["var_current"] * np.maximum(gpr, 1), minlength=T)
        dc = {"var_accelerator_type": acc_type, "var_gpus_per_replica": gpr,
              "mod_scale_to_zero_enabled": (g.random(M) < 0.3).astype(np.uint8),
              "mod_request_count": np.where(g.random(M) < 0.5, 0.0, 10.0), "mod_request_error": (g.random(M) < 0.05).astype(np.uint8),
              "type_limit": (used + g.integers(0, 400, T)).astype(np.int32), "enable_limiter": np.array([1], np.int32)}
        res = {}
        for name in (("graph", "graph_host_limit") if b % 2 == 0 else ("graph_host_limit", "graph")):
            t0 = time.perf_counter()
            res[name] = (run_new if name == "graph" else run_old)(d, slots, kvs, qs, dc)
            lat[name].append((time.perf_counter() - t0) * 1e3)
        for k in res["graph"]:
            assert np.array_equal(res["graph"][k], res["graph_host_limit"][k]), (b, k)
        decided.append(int(res["graph"]["has_decision"].sum()))
    new.close(); old.close()
    out = {"variants": int(V), "pods": S, "types": T, "decisions_per_batch_p50": int(np.median(decided)),
           "final_decisions_equal": True}
    for name, v in lat.items():
        v = np.array(v[4:])
        out[name] = {"p50_ms": float(np.percentile(v, 50)), "p99_ms": float(np.percentile(v, 99))}
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


if __name__ == "__main__":
    with pkg.Engine(0) as e:
        out = {"card": card(), "models_per_batch": M, "batches": B, "response_in_registry_order": measure(e, M, B, False),
               "response_shuffled": measure(e, M, B, True), "final_decisions": measure_decisions(e, M, B),
               "note": "batch arrival -> decisions: columnar write of two pod-keyed vectors (slot, value) + per-variant state + "
                       "per-model config into the page-locked arena, ONE CUDA graph launch (H2D, pack, V1 saturation analysis + "
                       "targets, D2H), limiter (wva_limit) on the host-visible results"}
    print(json.dumps(out))
