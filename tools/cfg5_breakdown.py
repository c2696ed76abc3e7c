import importlib, os, sys, time, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("llm-d-workload-variant-autoscaler_b200")
with pkg.Engine(0) as e:
    rows=[]
    for b in range(12):
        d = pkg.synth.saturation_batch(10_000, 32, stream=500 + b)
        t0=time.perf_counter(); r = e.saturation_v1(d); t1=time.perf_counter(); ts=e.timing()
        lim_in = {"n_types": 8, "acc_type": (np.arange(d["n_variants"]) % 8).astype(np.int32), "current": d["var_current"],
                  "target": np.maximum(r["var_target"], 0).astype(np.int32), "gpus_per_replica": np.ones(d["n_variants"], np.int32),
                  "spare": np.repeat(r["mod_avg_spare_kv"], 32), "cost": d["var_cost"], "type_limit": np.full(8, int(d["var_current"].sum() // 8 + 500), np.int32)}
        t2=time.perf_counter(); e.limit(lim_in); t3=time.perf_counter(); tl=e.timing()
        rows.append((1e3*(t1-t0), ts["h2d_ms"], ts["saturation_ms"], ts["d2h_ms"], 1e3*(t2-t1), 1e3*(t3-t2), tl["limit_ms"]))
    a=np.array(rows[3:]); print("sat_call_wall h2d sat_kernel d2h  py_between  limit_call_wall limit_dev")
    print(np.round(np.median(a,axis=0),3))
