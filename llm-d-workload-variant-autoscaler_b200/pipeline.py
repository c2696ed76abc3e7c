"""Host-side mirrors of the two pipeline interfaces the hot path sits behind, above the C-ABI.

* `SaturationAnalyzer` = `interfaces.SaturationAnalyzer` (internal/interfaces/saturation_analyzer.go:246-267), the V1
  percentage analyzer of internal/saturation/analyzer.go;
* `Limiter` = `pipeline.Limiter` (internal/engines/pipeline/limiter_interfaces.go:72-80) as `DefaultLimiter` with
  `TypeInventory` + `GreedyBySaturation` implements it (default_limiter.go:42-113).

Records are plain dicts carrying the reference's Go field names (`PodName`, `KvCacheUsage`, `QueueLength`,
`VariantName`, `AcceleratorName`, `Cost`; `VariantName`/`CurrentReplicas`/`DesiredReplicas`/`PendingReplicas`;
`TargetReplicas`, `GPUsPerReplica`, `SpareCapacity`, `GPUsAllocated`, `WasLimited`, `LimitedBy`, `DecisionSteps`), so a
case from analyzer_test.go / default_limiter_test.go transcribes field by field.  Python twin of
`go/wvab200/wvab200.go`; grouping, ordering and strings only — the arithmetic is `wva_saturation_v1` / `wva_limit`.
`ingest_decisions` is the string side of the ingest graph's decision mode (the whole optimizeV1 tail on the device).
"""
from __future__ import annotations

import numpy as np

SAT_SCALE_UP, SAT_SCALE_DOWN_SAFE = 1, 2


def _config(cfg: dict):
    g = lambda k: float(cfg.get(k, 0.0))
    return g("KvCacheThreshold"), g("QueueLengthThreshold"), g("KvSpareTrigger"), g("QueueSpareTrigger")


def scale_up_reason(avg_kv: float, avg_q: float, kv_trigger: float, q_trigger: float) -> str:
    """analyzer.go:199-225 (strings only; the flag itself comes from the device)."""
    kv_t, q_t = avg_kv < kv_trigger, avg_q < q_trigger
    if kv_t and q_t:
        return "both KV spare (%.3f < %.3f) and queue spare (%.1f < %.1f)" % (avg_kv, kv_trigger, avg_q, q_trigger)
    if kv_t:
        return "KV spare Saturation low (%.3f < %.3f)" % (avg_kv, kv_trigger)
    if q_t:
        return "queue spare Saturation low (%.1f < %.1f)" % (avg_q, q_trigger)
    return ""


class SaturationAnalyzer:
    """AnalyzeModelSaturation / CalculateSaturationTargets for one model per call, or `analyze_batch` for every model
    of a reconcile cycle in one launch (what the engine loop at engines/saturation/engine.go:779-795 would hoist)."""

    def __init__(self, engine):
        self.engine = engine

    # -- batching: variants ascending by name inside a model, replica order kept (sums are order dependent) ----
    @staticmethod
    def _pack(models):
        """models: list of (replica_metrics, config, variant_states|None) -> (SoA batch, per-model variant names,
        per-variant metrics lists)."""
        mvo, vro = [0], [0]
        kv, q, cost, cur, des, pen, has = [], [], [], [], [], [], []
        cfg4 = [[], [], [], []]
        names, groups = [], []
        for rm, cfg, states in models:
            by_var = {}
            for r in rm:
                by_var.setdefault(r["VariantName"], []).append(r)
            st = {s["VariantName"]: s for s in (states or [])}
            vnames = sorted(set(by_var) | set(st))        # a state without metrics is still a variant of the model
            for v in vnames:
                ms = by_var.get(v, [])
                kv += [float(r["KvCacheUsage"]) for r in ms]
                q += [int(r["QueueLength"]) for r in ms]
                vro.append(len(kv))
                cost.append(float(ms[0].get("Cost", 0.0)) if ms else 0.0)    # analyzer.go:146-148: first replica's cost
                s = st.get(v)
                cur.append(int(s["CurrentReplicas"]) if s else 0)
                des.append(int(s.get("DesiredReplicas", 0)) if s else 0)
                pen.append(int(s.get("PendingReplicas", 0)) if s else 0)
                has.append(1 if s else 0)
            mvo.append(len(vro) - 1)
            for i, c in enumerate(_config(cfg)):
                cfg4[i].append(c)
            names.append(vnames)
            groups.append(by_var)
        d = dict(n_models=len(models), n_variants=len(vro) - 1, n_replicas=len(kv), model_variant_off=mvo,
                 variant_replica_off=vro, rep_kv=kv, rep_queue=q, var_cost=cost, var_current=cur, var_desired=des,
                 var_pending=pen, var_has_state=has, cfg_kv_threshold=cfg4[0], cfg_queue_threshold=cfg4[1],
                 cfg_kv_trigger=cfg4[2], cfg_queue_trigger=cfg4[3])
        return d, names, groups

    def analyze_batch(self, models):
        """-> list of (ModelSaturationAnalysis dict, targets dict) in input order; one device launch."""
        models = list(models)
        if not models:
            return []
        d, names, groups = self._pack([(m["replicaMetrics"], m["config"], m.get("variantStates")) for m in models])
        out = self.engine.saturation_v1(d)
        res = []
        for mi, m in enumerate(models):
            cfg = _config(m["config"])
            flags = int(out["mod_flags"][mi])
            an = {"ModelID": m.get("modelID", ""), "Namespace": m.get("namespace", ""),
                  "TotalReplicas": int(out["mod_total_replicas"][mi]),
                  "NonSaturatedCount": int(out["mod_non_saturated"][mi]),
                  "AvgSpareKvCapacity": float(out["mod_avg_spare_kv"][mi]),
                  "AvgSpareQueueLength": float(out["mod_avg_spare_queue"][mi]),
                  "ShouldScaleUp": bool(flags & SAT_SCALE_UP), "ScaleUpReason": "",
                  "ScaleDownSafe": bool(flags & SAT_SCALE_DOWN_SAFE), "VariantAnalyses": []}
            if an["ShouldScaleUp"]:
                an["ScaleUpReason"] = scale_up_reason(an["AvgSpareKvCapacity"], an["AvgSpareQueueLength"], cfg[2], cfg[3])
            targets = {}
            v0 = d["model_variant_off"][mi]
            for k, v in enumerate(names[mi]):
                vi = v0 + k
                ms = groups[mi].get(v, [])
                if ms:
                    r0, r1 = d["variant_replica_off"][vi], d["variant_replica_off"][vi + 1]
                    an["VariantAnalyses"].append({
                        "VariantName": v, "AcceleratorName": ms[0].get("AcceleratorName", ""),
                        "Cost": float(d["var_cost"][vi]), "ReplicaCount": int(out["var_replica_count"][vi]),
                        "NonSaturatedCount": int(out["var_non_saturated"][vi]),
                        "MaxKvCacheUsage": float(out["var_max_kv"][vi]), "MaxQueueLength": int(out["var_max_queue"][vi]),
                        "AvgSpareKvCapacity": float(out["var_avg_spare_kv"][vi]),
                        "AvgSpareQueueLength": float(out["var_avg_spare_queue"][vi]),
                        "SaturatedReplicas": [ms[j - r0].get("PodName", "") for j in range(r0, r1) if out["rep_saturated"][j]]})
                if int(out["var_target"][vi]) >= 0:
                    targets[v] = int(out["var_target"][vi])
            res.append((an, targets))
        return res

    def analyze_model_saturation(self, model_id, namespace, replica_metrics, config):
        """AnalyzeModelSaturation (analyzer.go:29-133).  No metrics -> the empty analysis of analyzer.go:39-50."""
        if not replica_metrics:
            return {"ModelID": model_id, "Namespace": namespace, "TotalReplicas": 0, "NonSaturatedCount": 0,
                    "AvgSpareKvCapacity": 0.0, "AvgSpareQueueLength": 0.0, "ShouldScaleUp": False, "ScaleUpReason": "",
                    "ScaleDownSafe": False, "VariantAnalyses": [], "_src": ([], dict(config))}
        an, _ = self.analyze_batch([{"modelID": model_id, "namespace": namespace, "replicaMetrics": replica_metrics,
                                     "config": config}])[0]
        an["_src"] = (list(replica_metrics), dict(config))   # the device computes analysis + targets in one pass
        return an

    def calculate_saturation_targets(self, analysis, variant_states):
        """CalculateSaturationTargets (analyzer.go:296-420): map VariantName -> target replicas."""
        rm, cfg = analysis["_src"]
        if not rm:      # no analyses: every state keeps its current replicas (analyzer.go:303-320 loop over states)
            return {s["VariantName"]: int(s["CurrentReplicas"]) for s in variant_states} if variant_states else {}
        _, targets = self.analyze_batch([{"modelID": analysis["ModelID"], "namespace": analysis["Namespace"],
                                          "replicaMetrics": rm, "config": cfg, "variantStates": variant_states}])[0]
        return targets


class Limiter:
    """DefaultLimiter: `limits` is TypeInventory.limitByType after Refresh (type_inventory.go), a dict accelerator
    type -> GPUs, or a callable returning it.  `limit(decisions)` mutates the decisions in place
    (default_limiter.go:42-113): TargetReplicas, GPUsAllocated, WasLimited, LimitedBy, and one DecisionStep each."""

    def __init__(self, engine, name, limits):
        self.engine, self._name, self._limits = engine, name, limits

    def name(self):
        return self._name

    @staticmethod
    def _reason(d):
        ch = d["TargetReplicas"] - d["CurrentReplicas"]
        if ch <= 0:
            return "no scale-up (target=%d, current=%d)" % (d["TargetReplicas"], d["CurrentReplicas"])
        if d["WasLimited"]:
            return "limited: allocated %d GPUs for +%d replicas" % (d["GPUsAllocated"], ch)
        return "allocated %d GPUs for +%d replicas" % (d["GPUsAllocated"], ch)

    def limit(self, decisions):
        if not decisions:
            return
        lim = self._limits() if callable(self._limits) else self._limits
        types = sorted(lim)
        of = {t: i for i, t in enumerate(types)}
        acc_type = [of[d["AcceleratorName"]] if d.get("AcceleratorName", "") in of and d.get("AcceleratorName", "") != ""
                    else -1 for d in decisions]       # "" or a type without a pool: nothing can be allocated
        out = self.engine.limit({
            "n_types": len(types), "acc_type": acc_type,
            "current": [int(d["CurrentReplicas"]) for d in decisions], "target": [int(d["TargetReplicas"]) for d in decisions],
            "gpus_per_replica": [int(d.get("GPUsPerReplica", 0)) for d in decisions],
            "spare": [float(d.get("SpareCapacity", 0.0)) for d in decisions],
            "cost": [float(d.get("Cost", 0.0)) for d in decisions],
            "type_limit": np.array([int(lim[t]) for t in types], np.int32).reshape(-1)})
        for i, d in enumerate(decisions):
            d["TargetReplicas"] = int(out["target"][i])
            d["GPUsAllocated"] = int(out["gpus_allocated"][i])
            d["WasLimited"] = bool(out["was_limited"][i])
            if d["WasLimited"]:
                d["LimitedBy"] = self._name
            d.setdefault("DecisionSteps", []).append({"Name": self._name, "Action": d.get("Action", ""),
                                                      "TargetReplicas": d["TargetReplicas"], "Reason": self._reason(d),
                                                      "WasConstrained": d["WasLimited"]})


ACTION_NAMES = {1: "scale-up", -1: "scale-down", 0: "no-change"}     # interfaces.SaturationAction (saturation_analyzer.go:222-224)


def ingest_decisions(ing, models, variant_names, accelerator_names, limiter_name="gpu-limiter"):
    """The tail of optimizeV1 (engines/saturation/engine.go:322-392) as VariantDecision dicts, from a decision-mode
    `Ingest` after `commit()`: the device ran EnforcePolicy, convertSaturationTargetsToDecisions (:589-661) and the GPU
    limiter; this attaches the strings.  models: [(ModelID, Namespace)] per registry model; variant_names /
    accelerator_names: per registry variant (the AcceleratorName of the variant's analysis — read only for variants
    that reported, the others carry "" as `va == nil` does, :647-655).  `limiter_name` = the DefaultLimiter's name
    (engine.go:113).  Decisions come in registry order (the reference appends them per model in map order)."""
    r, d, c, cols = ing.res, ing.dres, ing.dcols, ing.cols
    mvo = np.asarray(ing.model_variant_off)
    limited_on = bool(c["enable_limiter"][0])
    out = []
    for v in np.flatnonzero(d["has_decision"]):
        v = int(v)
        m = int(np.searchsorted(mvo, v, side="right")) - 1
        va = int(r["var_replica_count"][v]) > 0
        g = int(c["var_gpus_per_replica"][v])
        action = ACTION_NAMES[int(d["action"][v])]
        dec = {"VariantName": variant_names[v], "ModelID": models[m][0], "Namespace": models[m][1],
               "CurrentReplicas": int(cols["var_current"][v]), "TargetReplicas": int(d["target"][v]),
               "OriginalTargetReplicas": int(d["original_target"][v]), "DesiredReplicas": int(cols["var_desired"][v]),
               "Action": action, "Reason": "saturation-only mode: " + action, "GPUsPerReplica": g if g > 0 else 1,
               "AcceleratorName": accelerator_names[v] if va else "", "Cost": float(cols["var_cost"][v]) if va else 0.0,
               "SpareCapacity": float(r["var_avg_spare_kv"][v]) if va else 0.0,
               "GPUsAllocated": int(d["gpus_allocated"][v]), "WasLimited": bool(d["was_limited"][v]), "LimitedBy": "",
               "DecisionSteps": []}
        if limited_on:                                # DefaultLimiter.updateDecisionMetadata (default_limiter.go:85-97)
            if dec["WasLimited"]:
                dec["LimitedBy"] = limiter_name
            dec["DecisionSteps"].append({"Name": limiter_name, "Action": action, "TargetReplicas": dec["TargetReplicas"],
                                         "Reason": Limiter._reason(dec), "WasConstrained": dec["WasLimited"]})
        out.append(dec)
    return out


# ======================================================================================================================
# V2 pipeline: token-capacity analyzer -> cost-aware optimizer -> enforcer (SURVEY §8f.1-2)
# ======================================================================================================================
ROLLING_AVERAGE_WINDOW = 10        # saturation_v2/constants.go RollingAverageWindowSize
SHORT_OUTPUT, MEDIUM_OUTPUT = 100, 500
COMPAT_FIELDS = ("GpuMemoryUtilization", "BlockSize", "KvCacheDtype", "TensorParallelSize", "NumGpuBlocksOverride",
                 "EffectiveMaxBatchedTokens")   # VLLMEngineParams.IsCapacityCompatible (deployment_parser.go:225-235)


def classify_output_length(avg_output: float) -> str:
    """types.go:28-37"""
    return "short" if avg_output < SHORT_OUTPUT else ("medium" if avg_output < MEDIUM_OUTPUT else "long")


def _go_int(x: float) -> int:
    """float64 -> int64 as Go on amd64"""
    if not (-9223372036854775808.0 <= x < 9223372036854775808.0):
        return -(1 << 63)
    return int(x)


def estimate_capacity_from_params(params, avg_in: float, avg_out: float) -> int:
    """estimateCapacityFromParams (analyzer.go:418-437) — part of the caller-side k2 chain, float64 as in Go."""
    if not params or params.get("EffectiveMaxBatchedTokens", 0) <= 0 or avg_out <= 0:
        return 0
    B, S = float(params["EffectiveMaxBatchedTokens"]), float(params.get("MaxNumSeqs", 0))
    n = B * avg_out / (avg_in + avg_out)
    if n > S:
        n = S
    k2 = _go_int(n * (avg_in + avg_out / 2))
    return k2 if k2 > 0 else 0


class CapacityKnowledgeStore:
    """capacity_store.go: records keyed namespace|model|variant (insertion order = Go map stand-in for FindCompatible)."""

    def __init__(self):
        self.records = {}

    def get(self, ns, model, variant):
        return self.records.get((ns, model, variant))

    def update(self, ns, model, variant, rec):
        self.records[(ns, model, variant)] = dict(rec)

    def find_compatible(self, model, accelerator, gpu_count, params):
        best = None
        for (ns, m, v), rec in self.records.items():
            if m != model or rec.get("AcceleratorName") != accelerator or rec.get("GpuCount") != gpu_count:
                continue
            p = rec.get("VLLMParams")
            if not p or not params or any(p.get(f) != params.get(f) for f in COMPAT_FIELDS):
                continue
            if rec.get("EffectiveCapacity", 0) <= 0 and rec.get("TotalKvCapacityTokens", 0) <= 0:
                continue
            if best is None or (best.get("LearnedFrom") != "live" and rec.get("LearnedFrom") == "live"):
                best = rec
        return best


class SaturationAnalyzerV2:
    """interfaces.Analyzer as saturation_v2.SaturationAnalyzer implements it (analyzer.go).  What the reference keeps in
    string-keyed state stays here, exactly as there — the rolling k2 history with its priority chain (computeK2
    :218-262), the capacity store and the zero-replica estimates (:317-324, :351-415) — and feeds the device the
    per-replica k2 and per-variant fallback capacity; all arithmetic on the metrics is `wva_saturation_v2`."""

    def __init__(self, engine, store: CapacityKnowledgeStore | None = None):
        self.engine = engine
        self.store = store or CapacityKnowledgeStore()
        self.history = {}          # "model|accelerator|bucket" -> list of float (window 10)

    def name(self):
        return "saturation-token-based"

    # -- caller-side state machines -----------------------------------------------------------------------------------
    def _k2(self, model_id, rm, queue_threshold, params):
        key = "%s|%s|%s" % (model_id, rm.get("AcceleratorName", ""), classify_output_length(float(rm.get("AvgOutputTokens", 0.0))))
        q, used = int(rm.get("QueueLength", 0)), int(rm.get("TokensInUse", 0))
        if q >= _go_int(queue_threshold) and used > 0:                      # priority 1: observed
            h = self.history.setdefault(key, [])
            if len(h) >= ROLLING_AVERAGE_WINDOW:
                del h[0]
            h.append(float(used))
            return used
        h = self.history.get(key)
        if h:                                                               # priority 2: rolling average
            s = 0.0
            for x in h:
                s += x
            avg = s / float(len(h))
            if avg > 0:
                return _go_int(avg)
        d = estimate_capacity_from_params(params, float(rm.get("AvgInputTokens", 0.0)), float(rm.get("AvgOutputTokens", 0.0)))
        return d if d > 0 else -1                                           # priority 3 / 4 (-1 = k1, known on the device)

    def _stored_capacity(self, rec, model_id, kv_thr, avg_in, avg_out):
        """estimateStoredCapacity (analyzer.go:365-415)"""
        if rec.get("LearnedFrom") == "live":
            return float(rec.get("EffectiveCapacity", 0))
        p = rec.get("VLLMParams")
        if p and avg_out > 0:
            derived = estimate_capacity_from_params(p, avg_in, avg_out)
            if derived > 0:
                bounded = derived
                if rec.get("TotalKvCapacityTokens", 0) > 0 and kv_thr > 0:
                    k1 = _go_int(float(rec["TotalKvCapacityTokens"]) * kv_thr)
                    if 0 < k1 < bounded:
                        bounded = k1
                c = self.store.find_compatible(model_id, rec.get("AcceleratorName"), rec.get("GpuCount"), p)
                if c is not None and c.get("LearnedFrom") == "live" and c.get("EffectiveCapacity", 0) > 0 and c["EffectiveCapacity"] < bounded:
                    bounded = c["EffectiveCapacity"]
                return float(bounded)
        return float(rec.get("EffectiveCapacity", 0))

    # -- Analyze ------------------------------------------------------------------------------------------------------
    def analyze(self, inp: dict) -> dict:
        """AnalyzerInput {ModelID, Namespace, ReplicaMetrics, VariantStates, Config, SchedulerQueue} -> AnalyzerResult."""
        return self.analyze_batch([inp])[0]

    def analyze_batch(self, inputs):
        mvo, vro = [0], [0]
        rep = {k: [] for k in ("tk", "tu", "ql", "ai", "ao", "hr", "k2")}
        order, vcur, vpen, vfb, cfg = [], [], [], [], ([], [], [])
        qs, qb, any_queue = [], [], False
        meta = []
        for inp in inputs:
            model, ns, c = inp.get("ModelID", ""), inp.get("Namespace", ""), inp["Config"]
            rms, states = inp.get("ReplicaMetrics", []) or [], inp.get("VariantStates", []) or []
            gpus = {s["VariantName"]: int(s.get("GPUsPerReplica", 0)) for s in states}
            kv_thr = float(c.get("KvCacheThreshold", 0.0))
            # phase 1 in slice order: the k2 chain mutates the history, the store is updated with live data
            k2_of, eff_of = {}, {}
            for i, rm in enumerate(rms):
                if int(rm.get("TotalKvCapacityTokens", 0)) <= 0:
                    continue
                rec = self.store.get(ns, model, rm["VariantName"])
                params = rec.get("VLLMParams") if rec else None
                k2_of[i] = self._k2(model, rm, float(c.get("QueueLengthThreshold", 0.0)), params)
            base = vro[-1]
            by_var = {}
            for i, rm in enumerate(rms):
                by_var.setdefault(rm["VariantName"], []).append(i)
            names = [s["VariantName"] for s in states]
            pos_of = {}
            for s in states:
                for i in by_var.get(s["VariantName"], []):
                    pos_of[i] = len(rep["tk"])
                    rep["tk"].append(int(rms[i].get("TotalKvCapacityTokens", 0))); rep["tu"].append(int(rms[i].get("TokensInUse", 0)))
                    rep["ql"].append(int(rms[i].get("QueueLength", 0))); rep["ai"].append(float(rms[i].get("AvgInputTokens", 0.0)))
                    rep["ao"].append(float(rms[i].get("AvgOutputTokens", 0.0))); rep["hr"].append(float(rms[i].get("PrefixCacheHitRate", 0.0)))
                    rep["k2"].append(int(k2_of.get(i, -1)))
                vro.append(len(rep["tk"]))
                vcur.append(int(s.get("CurrentReplicas", 0))); vpen.append(int(s.get("PendingReplicas", 0)))
            # replicas of variants without a state do not reach any VariantCapacity but count in the workload averages:
            # keep them in the slice order with a trailing phantom variant only if needed (not produced by the collector)
            order += [pos_of[i] for i in range(len(rms)) if i in pos_of]
            # per-model context for the zero-replica fallbacks, resolved after the live capacities reached the store
            ai = ao = 0.0; cnt = 0                                  # computeModelWorkloadAverages :438-455
            for rm in rms:
                if float(rm.get("AvgInputTokens", 0.0)) > 0 or float(rm.get("AvgOutputTokens", 0.0)) > 0:
                    ai += float(rm.get("AvgInputTokens", 0.0)); ao += float(rm.get("AvgOutputTokens", 0.0)); cnt += 1
            if cnt:
                ai /= float(cnt); ao /= float(cnt)
            accel = {}
            cost = {}
            for rm in rms:
                accel.setdefault(rm["VariantName"], rm.get("AcceleratorName", "")); cost.setdefault(rm["VariantName"], float(rm.get("Cost", 0.0)))
            vfb += [0.0] * len(states)
            avg_of = (ai, ao)
            mvo.append(len(vcur))
            cfg[0].append(kv_thr); cfg[1].append(float(c.get("ScaleUpThreshold", 0.0))); cfg[2].append(float(c.get("ScaleDownBoundary", 0.0)))
            sq = inp.get("SchedulerQueue")
            any_queue = any_queue or sq is not None
            qs.append(int(sq["QueueSize"]) if sq else 0); qb.append(int(sq["QueueBytes"]) if sq else 0)
            meta.append((inp, names, by_var, accel, cost, gpus, avg_of))
        d = dict(n_models=len(inputs), n_variants=len(vcur), n_replicas=len(rep["tk"]), model_variant_off=mvo, variant_replica_off=vro,
                 rep_total_kv_tokens=rep["tk"], rep_tokens_in_use=rep["tu"], rep_queue_length=rep["ql"], rep_avg_input_tokens=rep["ai"],
                 rep_avg_output_tokens=rep["ao"], rep_prefix_hit_rate=rep["hr"], rep_k2=rep["k2"], rep_slice_order=order,
                 var_current=vcur, var_pending=vpen, var_fallback_capacity=vfb, cfg_kv_threshold=cfg[0], cfg_scale_up_threshold=cfg[1],
                 cfg_scale_down_boundary=cfg[2], sched_queue_size=qs if any_queue else None, sched_queue_bytes=qb if any_queue else None)
        out = self.engine.saturation_v2(d)
        # the live capacities go into the store (analyzer.go:184-196, VLLMParams preserved) ...
        for mi, (inp, names, by_var, accel, cost, gpus, avg_of) in enumerate(meta):
            rms = inp.get("ReplicaMetrics", []) or []
            ns, model = inp.get("Namespace", ""), inp.get("ModelID", "")
            for k, v in enumerate(names):
                vi = mvo[mi] + k
                for j, i in enumerate(by_var.get(v, [])):
                    if int(rms[i].get("TotalKvCapacityTokens", 0)) > 0:
                        old = self.store.get(ns, model, v)
                        self.store.update(ns, model, v, {"AcceleratorName": rms[i].get("AcceleratorName", ""), "GpuCount": gpus.get(v, 0),
                                                         "NumGpuBlocks": int(rms[i].get("NumGpuBlocks", 0)), "BlockSize": int(rms[i].get("BlockSize", 0)),
                                                         "TotalKvCapacityTokens": int(rms[i]["TotalKvCapacityTokens"]),
                                                         "EffectiveCapacity": int(out["rep_effective"][vro[vi] + j]),
                                                         "VLLMParams": old.get("VLLMParams") if old else None, "LearnedFrom": "live"})
        # ... before the variants without ready replicas look a capacity up (:317-324); those models are evaluated again
        any_fb = False
        for mi, (inp, names, by_var, accel, cost, gpus, avg_of) in enumerate(meta):
            rms, states = inp.get("ReplicaMetrics", []) or [], inp.get("VariantStates", []) or []
            ns, model, kv_thr = inp.get("Namespace", ""), inp.get("ModelID", ""), cfg[0][mi]
            for k, st_ in enumerate(states):
                v = st_["VariantName"]
                if any(int(rms[i].get("TotalKvCapacityTokens", 0)) > 0 for i in by_var.get(v, [])):
                    continue
                fb, rec = 0.0, self.store.get(ns, model, v)
                if rec is not None and rec.get("EffectiveCapacity", 0) > 0:
                    fb = self._stored_capacity(rec, model, kv_thr, avg_of[0], avg_of[1])
                elif rec is not None and rec.get("VLLMParams"):
                    c2 = self.store.find_compatible(model, accel.get(v, ""), int(st_.get("GPUsPerReplica", 0)), rec["VLLMParams"])
                    if c2 is not None:
                        fb = float(c2.get("EffectiveCapacity", 0))
                if fb:
                    vfb[mvo[mi] + k] = fb
                    any_fb = True
        if any_fb:
            d["var_fallback_capacity"] = vfb
            out = self.engine.saturation_v2(d)
        self.last_batch, self.last_out = d, out
        results = []
        for mi, (inp, names, by_var, accel, cost, gpus, avg_of) in enumerate(meta):
            rms = inp.get("ReplicaMetrics", []) or []
            ns, model = inp.get("Namespace", ""), inp.get("ModelID", "")
            vcs = []
            for k, v in enumerate(names):
                vi = mvo[mi] + k
                a = accel.get(v, "")
                vcs.append({"VariantName": v, "AcceleratorName": a, "Cost": cost.get(v, 0.0),
                            "ReplicaCount": int(out["var_ready"][vi]), "PendingReplicas": int(vpen[vi]),
                            "PerReplicaCapacity": float(out["var_per_replica_capacity"][vi]),
                            "TotalCapacity": float(out["var_total_capacity"][vi]), "TotalDemand": float(out["var_total_demand"][vi]),
                            "Utilization": float(out["var_utilization"][vi])})
            results.append({"AnalyzerName": self.name(), "ModelID": model, "Namespace": ns, "VariantCapacities": vcs,
                            "TotalSupply": float(out["mod_total_supply"][mi]), "TotalDemand": float(out["mod_total_demand"][mi]),
                            "Utilization": float(out["mod_utilization"][mi]), "RequiredCapacity": float(out["mod_required_capacity"][mi]),
                            "SpareCapacity": float(out["mod_spare_capacity"][mi])})
        return results


class CostAwareOptimizer:
    """pipeline.ScalingOptimizer as CostAwareOptimizer implements it (cost_aware_optimizer.go:39-197): requests are
    ModelScalingRequest dicts {ModelID, Namespace, Result (AnalyzerResult | None), VariantStates}; one launch for all."""

    def __init__(self, engine):
        self.engine = engine

    def name(self):
        return "cost-aware"

    def optimize(self, requests, constraints=None):
        mvo, req, spare, has, cur, cost, cap = [0], [], [], [], [], [], []
        rows = []
        for r in requests:
            res = r.get("Result")
            states = r.get("VariantStates", []) or []
            st = {s["VariantName"]: s for s in states}
            vcs = (res or {}).get("VariantCapacities", []) or []
            vc_of = {vc["VariantName"]: vc for vc in vcs}
            # index space = VariantCapacities slice order, then states the analyzer did not report (capacity 0)
            names = [vc["VariantName"] for vc in vcs] + [s["VariantName"] for s in states if s["VariantName"] not in vc_of]
            for n in names:
                vc = vc_of.get(n, {})
                cur.append(int(st.get(n, {}).get("CurrentReplicas", 0))); cost.append(float(vc.get("Cost", 0.0)))
                cap.append(float(vc.get("PerReplicaCapacity", 0.0)))
            mvo.append(len(cur)); has.append(1 if res is not None else 0)
            req.append(float((res or {}).get("RequiredCapacity", 0.0))); spare.append(float((res or {}).get("SpareCapacity", 0.0)))
            rows.append((r, names, st, vc_of))
        tgt = self.engine.cost_aware_optimize(dict(model_variant_off=mvo, mod_required_capacity=req, mod_spare_capacity=spare,
                                                   mod_has_result=has, var_current=cur, var_cost=cost, var_per_replica_capacity=cap))
        decisions = []
        for mi, (r, names, st, vc_of) in enumerate(rows):
            if r.get("Result") is None:
                continue
            for k, n in enumerate(names):
                if n not in st and int(tgt[mvo[mi] + k]) == 0:
                    continue                                   # a capacity without a state only enters targets when it is scaled
                t, c = int(tgt[mvo[mi] + k]), int(st.get(n, {}).get("CurrentReplicas", 0))
                if t > c:
                    action, reason = "scale-up", "V2 scale-up (optimizer: cost-aware, required: %.0f)" % r["Result"].get("RequiredCapacity", 0.0)
                elif t < c:
                    action, reason = "scale-down", "V2 scale-down (optimizer: cost-aware, spare: %.0f)" % r["Result"].get("SpareCapacity", 0.0)
                else:
                    action, reason = "no-change", "V2 steady state"
                vc = vc_of.get(n, {})
                decisions.append({"VariantName": n, "ModelID": r.get("ModelID", ""), "Namespace": r.get("Namespace", ""),
                                  "AcceleratorName": vc.get("AcceleratorName", ""), "Cost": float(vc.get("Cost", 0.0)),
                                  "CurrentReplicas": c, "TargetReplicas": t, "Action": action, "Reason": reason})
        return decisions


class Enforcer:
    """pipeline.Enforcer (enforcer.go:55-183).  request_count_func(model_id, namespace, retention) -> float, may raise."""

    def __init__(self, engine, request_count_func):
        self.engine, self.request_count_func = engine, request_count_func

    def enforce_policy(self, model_id, namespace, saturation_targets: dict, variant_analyses, scale_to_zero_enabled: bool,
                       retention_period=None):
        names = sorted(saturation_targets)                     # the tie-break compares names: index order = name order
        cost_of = {va["VariantName"]: float(va.get("Cost", 0.0)) for va in (variant_analyses or [])}
        count, err = 0.0, 0
        if scale_to_zero_enabled:
            try:
                count = float(self.request_count_func(model_id, namespace, retention_period))
            except Exception:                                  # "Failed to get request count, keeping current targets"
                err = 1
        tgt, app = self.engine.enforce(dict(model_variant_off=[0, len(names)], mod_scale_to_zero_enabled=[1 if scale_to_zero_enabled else 0],
                                            mod_request_count=[count], mod_request_error=[err],
                                            var_cost=[cost_of.get(n, 0.0) for n in names], var_has_cost=[1 if n in cost_of else 0 for n in names],
                                            var_target=[int(saturation_targets[n]) for n in names]))
        for i, n in enumerate(names):
            saturation_targets[n] = int(tgt[i])
        return saturation_targets, bool(app[0])
