"""Time wva_k2_resolve (the V2 k2 priority chain with its rolling history in HBM) on a perf_v2.py-shaped cycle:
M model groups x 32 variants x 1..8 replicas, 1-3 namespaces per modelID (history group), 2-4 accelerators per modelID,
about 30 % of the data replicas observed (queue >= threshold).  Reports the device time of the keys + resolve + slot
kernels (CUDA events inside the library, best of the timed cycles after warm-up), the algorithmic bytes and GB/s, the
wall time of the host chain it replaces (the single-thread oracle walk over the same inputs), and the card.
usage: python tools/perf_k2.py [M=200000] [cycles=5]"""
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
from tests.k2_oracle import K2Oracle  # noqa: E402

M = int(sys.argv[1]) if len(sys.argv) > 1 else 200000
CYCLES = int(sys.argv[2]) if len(sys.argv) > 2 else 5
g = np.random.default_rng(0xB2005EED)

# registry: history groups of 1-3 model groups (registry order = index order), 2-4 accelerators each
sizes = []
while sum(sizes) < M:
    sizes.append(int(min(g.integers(1, 4), M - sum(sizes))))
H = len(sizes)
hg_model_off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int32)
hg_models = np.arange(M, dtype=np.int32)
n_acc = g.integers(2, 5, H)
hg_acc_off = np.concatenate(([0], np.cumsum(n_acc))).astype(np.int32)
hg_acc = np.concatenate([g.choice(8, int(k), replace=False) for k in n_acc]).astype(np.int32)
S = M * 32
hg_of = np.repeat(np.arange(H), sizes)


def cycle():
    nr = g.integers(1, 9, S)                                         # replicas per variant (slot), variants of a group contiguous
    per_group = nr.reshape(M, 32).sum(1)
    off = np.concatenate(([0], np.cumsum(per_group))).astype(np.int32)
    P = int(off[-1])
    slot = np.repeat(np.arange(S, dtype=np.int32), nr)
    h = hg_of[slot // 32]
    var_acc = (g.random(S) * n_acc[hg_of[np.arange(S) // 32]]).astype(np.int64)   # one accelerator per variant
    acc = hg_acc[hg_acc_off[h] + var_acc[slot]]
    cap = g.choice([8000, 16000, 32000, 64000], P).astype(np.int64)
    return {"model_replica_off": off, "rep_total_kv_tokens": cap, "rep_tokens_in_use": (cap * g.uniform(0.01, 1.0, P)).astype(np.int64),
            "rep_queue_length": g.integers(0, 10, P), "rep_avg_input_tokens": g.uniform(10, 2000, P),
            "rep_avg_output_tokens": g.uniform(10, 800, P), "rep_accelerator": acc.astype(np.int32), "rep_slot": slot,
            "slot_max_batched_tokens": g.integers(0, 8192, S) * (g.random(S) < 0.5), "slot_max_num_seqs": g.integers(16, 512, S),
            "cfg_queue_threshold": np.full(M, 7.0), "cfg_kv_threshold": np.full(M, 0.8)}


cycles = [cycle() for _ in range(2 + CYCLES)]
P = len(cycles[-1]["rep_total_kv_tokens"])
K = 3 * int(hg_acc_off[-1])
observed = float(np.mean(cycles[-1]["rep_queue_length"] >= 7))
# algorithmic bytes of one cycle: replica inputs once (5 x 8 B metrics + 2 x 4 B ids) and two int64 outputs; per slot
# two int64 params and two outputs (4 + 8 B); per group offsets and two thresholds; every ring read and written once
alg_bytes = P * (5 * 8 + 2 * 4 + 2 * 8) + S * (16 + 12) + M * (4 + 16) + K * (10 * 8 + 8) * 2

res = {"M": M, "H": H, "P": P, "S": S, "keys": K, "observed_fraction": round(observed, 3)}
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30).stdout.strip().splitlines()
    res["card"] = q[0] if q else "unknown"
except (OSError, subprocess.SubprocessError):
    res["card"] = "unknown"

with pkg.Engine(0) as e, pkg.K2History(e, hg_model_off, hg_models, hg_acc_off, hg_acc, S) as dev:
    ts = []
    for k, c in enumerate(cycles):
        dev.resolve(c)
        if k >= 2:                                                   # the first two cycles warm up (and fill the rings)
            ts.append(e.timing()["saturation_ms"])
    best = min(ts)
    res["resolve_kernels_ms"] = round(best, 4)
    res["resolve_kernels_ms_all"] = [round(t, 4) for t in ts]
    res["alg_bytes"] = alg_bytes
    res["alg_GBs"] = round(alg_bytes / (best * 1e-3) / 1e9, 1)
    d_exp = dev.export()

orc = K2Oracle(hg_model_off, hg_models, hg_acc_off, hg_acc, S)
wall = []
for c in cycles:
    t0 = time.perf_counter()
    orc.resolve(c)
    wall.append(time.perf_counter() - t0)
res["host_chain_ms"] = round(min(wall[2:]) * 1e3, 1)
cnt, vals = orc.export()
res["device_history_equals_oracle"] = bool(np.array_equal(cnt, d_exp["count"]) and
                                           np.array_equal(vals.view(np.int64), d_exp["values"].view(np.int64)))
print(json.dumps(res))
