"""TEST INFRASTRUCTURE: a literal restatement of the reference's CollectReplicaMetrics join for the V2 fields
(internal/collector/replica_metrics.go:78-403) over MockPromAPI-shaped vectors (a list of samples, each a label dict +
value), and a seeded multi-cycle fleet generator that exercises every fold rule.

    collect(vectors, pod_to_variant, accelerator_of, cost_of, variant_rank) -> ReplicaMetrics dicts

Order: the reference appends in Go-map order; here (variant registry rank, PodName), the canonical order the product
uses.  Nothing in this module is imported by the product."""
from __future__ import annotations

import math
import re

import numpy as np

from tests.collector_ref import INT64_MIN, _pod, go_int

INT64_MAX = (1 << 63) - 1
VECTORS = ("kv", "queue", "cache_config", "avg_output", "avg_input", "hit_rate")


def parse_int64(s):
    """strconv.ParseInt(s, 10, 64): None on error"""
    if s is None or not re.fullmatch(r"[+-]?[0-9]+", s):
        return None
    x = int(s)
    return x if -(1 << 63) <= x <= INT64_MAX else None


def go_round(x: float) -> float:
    """math.Round: half away from zero (x - trunc(x) is exact in float64)"""
    if math.isnan(x) or math.isinf(x):
        return x
    t = float(math.trunc(x))
    if abs(x - t) >= 0.5:
        t += math.copysign(1.0, x)
    return t


def go_int64(x: float) -> int:
    """int64(float64) on amd64: NaN / out of range -> INT64_MIN"""
    if math.isnan(x) or not (-9223372036854775808.0 <= x < 9223372036854775808.0):
        return INT64_MIN
    return int(x)


def _wrap64(x: int) -> int:
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def tokens(blocks: int, size: int, kv: float):
    """TotalKvCapacityTokens and TokensInUse with hasCacheConfig (:351-369)"""
    if blocks > 0 and size > INT64_MAX // blocks:
        total = INT64_MAX
    else:
        total = _wrap64(blocks * size)
    r = go_round(kv * float(total))
    if r < 0:
        r = 0.0
    elif r > float(total):
        r = float(total)
    return total, go_int64(r)


def collect(vec, pod_to_variant, accelerator_of, cost_of, variant_rank):
    pod = {}

    def rec(labels):
        name = _pod(labels)
        return pod.setdefault(name, {}) if name else None
    for labels, value in vec["kv"]:                                  # :133-160
        d = rec(labels)
        if d is not None:
            d["kv"] = float(value); d["hasKv"] = True
    for labels, value in vec["queue"]:                               # :163-189
        d = rec(labels)
        if d is not None:
            d["queue"] = go_int(float(value)); d["hasQueue"] = True
    for labels, _ in vec["cache_config"]:                            # :192-225
        d = rec(labels)
        if d is None:
            continue
        b = parse_int64(labels.get("num_gpu_blocks")) if labels.get("num_gpu_blocks") else None
        s = parse_int64(labels.get("block_size")) if labels.get("block_size") else None
        if b is not None:
            d["blocks"] = b
        if s is not None:
            d["size"] = s
        if d.get("blocks", 0) > 0 and d.get("size", 0) > 0:
            d["hasCC"] = True
    for key, field, rate in (("avg_output", "ao", False), ("avg_input", "ai", False), ("hit_rate", "hr", True)):   # :228-292
        for labels, value in vec[key]:
            d = rec(labels)
            if d is None:
                continue
            x = float(value)
            if math.isfinite(x) and (not rate or 0 <= x <= 1):
                d[field] = x
    out = []
    for name, d in pod.items():                                      # :296-396
        if not d.get("hasKv") and not d.get("hasQueue"):
            continue
        va = pod_to_variant.get(name, "")
        if va == "":
            continue
        kv = d["kv"] if d.get("hasKv") else 0.0
        total, used = tokens(d.get("blocks", 0), d.get("size", 0), kv) if d.get("hasCC") else (0, 0)
        out.append({"PodName": name, "VariantName": va, "AcceleratorName": accelerator_of[va], "KvCacheUsage": kv,
                    "QueueLength": d["queue"] if d.get("hasQueue") else 0, "Cost": cost_of[va],
                    "NumGpuBlocks": d.get("blocks", 0), "BlockSize": d.get("size", 0), "TotalKvCapacityTokens": total,
                    "TokensInUse": used, "AvgOutputTokens": d.get("ao", 0.0), "AvgInputTokens": d.get("ai", 0.0),
                    "PrefixCacheHitRate": d.get("hr", 0.0)})
    out.sort(key=lambda r: (variant_rank[r["VariantName"]], r["PodName"]))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# seeded fleet: registry + cycles
# ---------------------------------------------------------------------------------------------------------------------
ACCS = ("H100", "A100", "L40S")


def fleet(n_models, max_variants, seed, n_ids=None, exact=False):
    """models (modelID shared by up to 3 namespaces), their variants (names not in name order, so the enforcer's
    name tie-break differs from the registry order) and pods; deployment params for some variants.  exact: every
    model has max_variants variants (else 1..max_variants)"""
    g = np.random.default_rng(seed)
    n_ids = n_ids or max(1, (n_models + 2) // 3)
    models, variants, pods = [], [], {}
    for m in range(n_models):
        models.append(("model-%d" % (m % n_ids), "ns-%d" % (m // n_ids)))
        nv = max_variants if exact else int(g.integers(1, max_variants + 1))
        names = ["v%02d-%s" % (int(k), "abc"[int(k) % 3]) for k in g.permutation(nv)]
        vs = []
        for n in names:
            full = "m%05d-%s" % (m, n)                         # unique in the fleet: pods map to it by name
            vs.append({"name": full, "acc": str(g.choice(ACCS)), "gpus": int(g.integers(1, 3)),
                       "cost": float(g.choice((1.0, 2.5, 10.0, 40.0)))})
            k = int(g.integers(0, 5))
            pods[(m, full)] = sorted("%s-%s-pod-%04x" % (models[-1][0], full, int(x)) for x in g.choice(65536, k, replace=False))
        variants.append(vs)
    # VLLMEngineParams per deployment: half drawn from a small pool per modelID, so that variants of one modelID in
    # different namespaces are capacity-compatible (FindCompatible finds them); some without EffectiveMaxBatchedTokens
    # (no deployment estimate: the fallback then looks for a compatible record), some with num_gpu_blocks_override
    def draw():
        emb = 0 if g.random() < 0.25 else int(g.integers(512, 8192))
        return {"EffectiveMaxBatchedTokens": emb, "MaxNumSeqs": int(g.integers(16, 512)), "BlockSize": int(g.choice((16, 32))),
                "NumGpuBlocksOverride": int(g.integers(500, 4000)) if g.random() < 0.4 else 0, "GpuMemoryUtilization": 0.9,
                "KvCacheDtype": "auto", "TensorParallelSize": 1}
    pool = {mid: [draw() for _ in range(2)] for mid in {m for m, _ in models}}
    params = {}
    for m, vs in enumerate(variants):
        for v in vs:
            if g.random() < 0.6:
                p = pool[models[m][0]][int(g.integers(0, 2))] if g.random() < 0.5 else draw()
                params[(models[m][1], models[m][0], v["name"])] = dict(p)
                if g.random() < 0.5:                              # the pool's accelerator / GPU count: compatible records
                    v["acc"], v["gpus"] = ACCS[0], 1
    cfg = []
    for m in range(n_models):
        cfg.append({"KvCacheThreshold": float(g.choice((0.8, 0.9, 0.5))), "QueueLengthThreshold": float(g.choice((5.0, 2.5, 0.0))),
                    "ScaleUpThreshold": float(g.choice((0.85, 0.7))), "ScaleDownBoundary": float(g.choice((0.7, 0.5, 0.0)))})
    return {"models": models, "variants": variants, "pods": pods, "params": params, "cfg": cfg}


def cycle(fl, seed):
    """one cycle: the six vectors (shuffled, with every case the fold distinguishes) and the per-cycle columns"""
    g = np.random.default_rng(seed)
    vec = {k: [] for k in VECTORS}
    silent = set(int(m) for m in np.flatnonzero(g.random(len(fl["models"])) < 0.1))
    for (m, va), names in fl["pods"].items():
        gone = m in silent or g.random() < 0.1                        # a variant with no reporting pod this cycle
        for p in names:
            lab = {"pod": p} if g.random() < 0.8 else {"pod_name": p}
            only_v2 = gone or g.random() < 0.05                       # no kv / queue sample: skipped however rich
            if not only_v2:
                r = g.random()
                if r > 0.05:
                    kv = float(g.beta(2.0, 3.0))
                    vec["kv"].append((dict(lab), kv))
                    if g.random() < 0.05:
                        vec["kv"].append((dict(lab), float(g.random())))             # duplicate: the later wins
                if r < 0.95:
                    q = float(g.poisson(3.0)) + (0.75 if g.random() < 0.05 else 0.0)
                    vec["queue"].append((dict(lab), q))
            c = g.random()
            if c < 0.75:
                blocks, size = str(int(g.integers(1000, 40000))), str(int(g.choice((16, 32))))
                if g.random() < 0.05:
                    blocks, size = str(1 << 40), str(1 << 30)                         # blocks * size overflows
                elif g.random() < 0.05:
                    blocks = "0"                                                      # zero: no cache config
                elif g.random() < 0.03:
                    blocks = "12x"                                                    # does not parse
                elif g.random() < 0.05:
                    blocks, size = "4096", "16"                                       # kv on a 1/(2 * 65536) grid: .5 ties
                    kv_tie = float(int(g.integers(0, 65536)) * 2 + 1) / (2 * 65536)
                    vec["kv"].append((dict(lab), kv_tie))
                vec["cache_config"].append(({**lab, "num_gpu_blocks": blocks, "block_size": size}, 1.0))
                if g.random() < 0.05:
                    vec["cache_config"].append(({**lab, "num_gpu_blocks": "", "block_size": "64"}, 1.0))   # label empty
            for key, lo, hi in (("avg_output", 0.0, 900.0), ("avg_input", 0.0, 1200.0), ("hit_rate", 0.0, 1.0)):
                if g.random() < 0.85:
                    vec[key].append((dict(lab), float(g.uniform(lo, hi))))
                    if g.random() < 0.08:
                        bad = (float("nan"), float("inf"), -float("inf")) + ((1.5, -0.25) if key == "hit_rate" else ())
                        vec[key].append((dict(lab), bad[int(g.integers(0, len(bad)))]))     # does not overwrite
            if g.random() < 0.03:
                vec["avg_output"].append((dict(lab), float(g.choice((99.999, 100.0, 499.999, 500.0)))))
    for k in VECTORS:
        vec[k].append(({"pod": "stray-%x" % int(g.integers(1 << 30))}, 0.5))         # an unknown pod
        vec[k].append(({}, 0.25))                                                  # no pod label
        vec[k] = [vec[k][i] for i in g.permutation(len(vec[k]))]    # both paths read the samples in this order
    V = sum(len(vs) for vs in fl["variants"])
    M = len(fl["models"])
    state = {"current": g.integers(0, 5, V).astype(np.int32), "pending": (g.random(V) < 0.1).astype(np.int32)}
    state["current"][g.random(V) < 0.1] = 0
    mod = {"s2z": (g.random(M) < 0.3).astype(np.uint8), "count": np.where(g.random(M) < 0.5, 0.0, g.uniform(1, 100, M)),
           "err": (g.random(M) < 0.1).astype(np.uint8)}
    return vec, state, mod


# ---------------------------------------------------------------------------------------------------------------------
# the integer registry of a fleet, a cycle written into an IngestV2, and the same cycle as the reference's inputs
# ---------------------------------------------------------------------------------------------------------------------
class Registry:
    """slots of a variant in ascending pod name; store slot = variant index; history group = modelID (its models in
    registry order, its accelerators in first-seen order)"""

    def __init__(self, fl):
        self.fl = fl
        self.mvo, self.vso, self.slot_of, self.var = [0], [0], {}, []     # var: (model index, variant dict)
        for m, vs in enumerate(fl["variants"]):
            for v in vs:
                self.var.append((m, v))
                for p in fl["pods"][(m, v["name"])]:
                    self.slot_of[p] = len(self.slot_of)
                self.vso.append(len(self.slot_of))
            self.mvo.append(len(self.var))
        self.mvo, self.vso = np.array(self.mvo, np.int32), np.array(self.vso, np.int32)
        self.acc_id = {a: i for i, a in enumerate(ACCS)}
        self.var_acc = np.array([self.acc_id[v["acc"]] for _, v in self.var], np.int32)
        self.var_slot = np.arange(len(self.var), dtype=np.int32)
        self.names = [v["name"] for _, v in self.var]
        self.rank = np.zeros(len(self.var), np.int32)
        for m in range(len(fl["models"])):
            lo, hi = int(self.mvo[m]), int(self.mvo[m + 1])
            for r, k in enumerate(sorted(range(lo, hi), key=lambda k: self.names[k])):
                self.rank[k] = r
        self.variant_rank = {n: i for i, n in enumerate(self.names)}
        self.pod_to_variant = {p: v["name"] for (m, vn), ps in fl["pods"].items() for p in ps for v in fl["variants"][m] if v["name"] == vn}
        hgs, accs = {}, {}
        for m, (mid, _) in enumerate(fl["models"]):
            hgs.setdefault(mid, []).append(m)
            for k in range(int(self.mvo[m]), int(self.mvo[m + 1])):
                accs.setdefault(mid, {})[int(self.var_acc[k])] = None
        self.hgs = list(hgs)
        self.hg_model_off = np.concatenate(([0], np.cumsum([len(hgs[h]) for h in self.hgs]))).astype(np.int32)
        self.hg_models = np.array([m for h in self.hgs for m in hgs[h]], np.int32)
        self.hg_acc_off = np.concatenate(([0], np.cumsum([len(accs[h]) for h in self.hgs]))).astype(np.int32)
        self.hg_acc = np.array([a for h in self.hgs for a in accs[h]], np.int32)
        self.n_store_slots = max(len(self.var), 1)

    def k2_registry(self):
        return self.hg_model_off, self.hg_models, self.hg_acc_off, self.hg_acc, self.n_store_slots

    def seed_store(self, store):
        """the deployment-derived records every path starts from, as CapacityKnowledgeStore.LoadFromDeployment makes
        them (capacity_store.go:88-124): k1 data from num_gpu_blocks_override, EffectiveCapacity =
        EffectiveMaxBatchedTokens when that is > 0"""
        for k, (m, v) in enumerate(self.var):
            mid, ns = self.fl["models"][m]
            p = self.fl["params"].get((ns, mid, v["name"]))
            if p:
                rec = {"AcceleratorName": v["acc"], "GpuCount": v["gpus"], "VLLMParams": p, "LearnedFrom": "deployment",
                       "NumGpuBlocks": 0, "BlockSize": 0, "TotalKvCapacityTokens": 0, "EffectiveCapacity": 0}
                if p["NumGpuBlocksOverride"] > 0:
                    rec.update(NumGpuBlocks=p["NumGpuBlocksOverride"], BlockSize=p["BlockSize"],
                               TotalKvCapacityTokens=p["NumGpuBlocksOverride"] * p["BlockSize"])
                if p["EffectiveMaxBatchedTokens"] > 0:
                    rec["EffectiveCapacity"] = p["EffectiveMaxBatchedTokens"]
                store.update(ns, mid, v["name"], rec)

    def slot_params(self, store):
        """per store slot: EffectiveMaxBatchedTokens, MaxNumSeqs of the record's VLLMParams at the cycle's start"""
        B, S = np.zeros(self.n_store_slots, np.int64), np.zeros(self.n_store_slots, np.int64)
        for k, (m, v) in enumerate(self.var):
            mid, ns = self.fl["models"][m]
            rec = store.get(ns, mid, v["name"])
            p = (rec.get("VLLMParams") if rec else None) or {}
            B[k], S[k] = int(p.get("EffectiveMaxBatchedTokens", 0)), int(p.get("MaxNumSeqs", 0))
        return B, S

    def slots(self, vector):
        return np.array([self.slot_of.get(_pod(lab), -1) for lab, _ in vector], np.int32), np.array([v for _, v in vector], np.float64)

    def write(self, ing, abi, vec, state, mod, store):
        """what the collector does each cycle: begin, the six vectors, the per-cycle columns"""
        ing.begin()
        for key, which in (("kv", abi.VEC_KV_CACHE_USAGE), ("queue", abi.VEC_QUEUE_LENGTH), ("avg_output", abi.VEC_AVG_OUTPUT_TOKENS),
                           ("avg_input", abi.VEC_AVG_INPUT_TOKENS), ("hit_rate", abi.VEC_PREFIX_CACHE_HIT_RATE)):
            ing.write(which, *self.slots(vec[key]))
        sl = self.slots(vec["cache_config"])[0]
        lab = lambda s: (parse_int64(s) if s else None)
        b = [lab(x.get("num_gpu_blocks")) for x, _ in vec["cache_config"]]
        z = [lab(x.get("block_size")) for x, _ in vec["cache_config"]]
        ing.write_cache_config(sl, [abi.CACHE_LABEL_ABSENT if x is None else x for x in b],
                               [abi.CACHE_LABEL_ABSENT if x is None else x for x in z])
        c = ing.cols
        c["var_cost"][:] = [v["cost"] for _, v in self.var]
        c["var_current"][:] = state["current"]; c["var_pending"][:] = state["pending"]; c["var_name_rank"][:] = self.rank
        cfg = self.fl["cfg"]
        c["cfg_kv_threshold"][:] = [x["KvCacheThreshold"] for x in cfg]
        c["cfg_queue_threshold"][:] = [x["QueueLengthThreshold"] for x in cfg]
        c["cfg_scale_up_threshold"][:] = [x["ScaleUpThreshold"] for x in cfg]
        c["cfg_scale_down_boundary"][:] = [x["ScaleDownBoundary"] for x in cfg]
        c["mod_scale_to_zero_enabled"][:] = mod["s2z"]; c["mod_request_count"][:] = mod["count"]
        c["mod_request_error"][:] = mod["err"]
        c["slot_max_batched_tokens"][:], c["slot_max_num_seqs"][:] = self.slot_params(store)

    def decisions_args(self):
        return (self.fl["models"], self.names, [v["acc"] for _, v in self.var], [v["gpus"] for _, v in self.var])

    def reference_inputs(self, vec, state, mod):
        """the cycle as optimizeV2 sees it: AnalyzerInputs of the models with a reporting pod, their scale-to-zero
        flags, and the request-count function (raises for the models whose query fails)"""
        recs = collect(vec, self.pod_to_variant, {v["name"]: v["acc"] for _, v in self.var},
                       {v["name"]: v["cost"] for _, v in self.var}, self.variant_rank)
        model_of = {v["name"]: m for m, v in self.var}
        per = {}
        for r in recs:
            per.setdefault(model_of[r["VariantName"]], []).append(r)
        inputs, s2z, counts = [], [], {}
        for m, (mid, ns) in enumerate(self.fl["models"]):
            if m not in per:
                continue                                   # prepareModelData returns nil: no request
            states = [{"VariantName": self.var[k][1]["name"], "CurrentReplicas": int(state["current"][k]),
                       "PendingReplicas": int(state["pending"][k]), "GPUsPerReplica": self.var[k][1]["gpus"]}
                      for k in range(int(self.mvo[m]), int(self.mvo[m + 1]))]
            inputs.append({"ModelID": mid, "Namespace": ns, "ReplicaMetrics": per[m], "VariantStates": states,
                           "Config": self.fl["cfg"][m], "SchedulerQueue": None})
            s2z.append(int(mod["s2z"][m]))
            counts[(mid, ns)] = None if mod["err"][m] else float(mod["count"][m])

        def count(model, ns, _retention):
            c = counts[(model, ns)]
            if c is None:
                raise RuntimeError("request count query failed")
            return c
        return inputs, s2z, count, per
