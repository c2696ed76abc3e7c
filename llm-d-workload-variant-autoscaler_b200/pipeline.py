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
BUCKETS = ("short", "medium", "long")     # output-length buckets, in the device history's bucket order
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
    """capacity_store.go: records keyed namespace|model|variant (insertion order = Go map stand-in for FindCompatible).
    Records are written through update() only: find_compatible visits a model's keys from an index update() keeps, so a
    record placed into `records` directly is not seen by it."""

    def __init__(self):
        self.records = {}
        self._of_model = {}        # model -> its keys in the records' insertion order (FindCompatible visits no other)

    def get(self, ns, model, variant):
        return self.records.get((ns, model, variant))

    def update(self, ns, model, variant, rec):
        self.records[(ns, model, variant)] = dict(rec)
        self._of_model.setdefault(model, {})[(ns, model, variant)] = None

    def find_compatible(self, model, accelerator, gpu_count, params):
        best = None
        for key in self._of_model.get(model, ()):
            rec = self.records[key]
            if rec.get("AcceleratorName") != accelerator or rec.get("GpuCount") != gpu_count:
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

    def __init__(self, engine, store: CapacityKnowledgeStore | None = None, device_history: bool = False):
        """device_history: keep the rolling k2 history on the device (`engine.K2History`) and resolve the k2 chain and
        the per-slot store updates there (`wva_k2_resolve`) instead of in the host chain below."""
        self.engine = engine
        self.store = store or CapacityKnowledgeStore()
        self.history = {}          # "model|accelerator|bucket" -> list of float (window 10); host chain only
        self.k2 = None             # the device history (device_history=True), rebuilt when its registry changes
        self.device_history = device_history
        self._k2_reg = None        # (modelID per input, {modelID: accelerator names}, n_slots) of self.k2
        self._k2_hgs = []          # modelID per history group of self.k2
        self._acc_id, self._slot = {}, {}   # accelerator name -> id; (namespace, model, variant) -> store slot

    def name(self):
        return "saturation-token-based"

    def close(self):
        if self.k2 is not None:
            self.k2.close()
            self.k2 = None

    # -- the device history -------------------------------------------------------------------------------------------
    def history_state(self) -> dict:
        """the rolling history as {"model|accelerator|bucket": [values oldest first]} (keys with values only)"""
        if not self.device_history:
            return {k: list(v) for k, v in self.history.items() if v}
        if self.k2 is None:
            return {}
        e, names = self.k2.export(), {i: n for n, i in self._acc_id.items()}
        return {"%s|%s|%s" % (self._k2_hgs[int(e["hg"][k])], names[int(e["acc"][k])], BUCKETS[int(e["bucket"][k])]):
                [float(x) for x in e["values"][k, :int(e["count"][k])]] for k in range(len(e["hg"])) if e["count"][k] > 0}

    def _k2_registry(self, inputs):
        """the handle for this batch: its model groups are the inputs in list order, its history groups every modelID of
        the batch and every modelID the history already holds.  A new registry = export, create, import."""
        models = tuple(inp.get("ModelID", "") for inp in inputs)
        accs = {}
        for m, inp in zip(models, inputs):
            for rm in inp.get("ReplicaMetrics", []) or []:
                accs.setdefault(m, {})[rm.get("AcceleratorName", "")] = None
                self._slot.setdefault((inp.get("Namespace", ""), m, rm["VariantName"]), len(self._slot))
            for s in inp.get("VariantStates", []) or []:
                self._slot.setdefault((inp.get("Namespace", ""), m, s["VariantName"]), len(self._slot))
        if self.k2 is not None and self._k2_reg[0] == models and len(self._slot) <= self._k2_reg[2] and \
                all(a in self._k2_reg[1].get(m, ()) for m, s in accs.items() for a in s):
            return
        old = self.history_state()
        for key in old:
            m, a, _ = key.rsplit("|", 2)
            accs.setdefault(m, {})[a] = None
        for m, s in (self._k2_reg[1] if self._k2_reg else {}).items():
            for a in s:
                accs.setdefault(m, {})[a] = None
        hgs = list(dict.fromkeys(models + tuple(accs)))
        mo, mg, ao, ai = [0], [], [0], []
        for m in hgs:
            mg += [i for i, x in enumerate(models) if x == m]
            mo.append(len(mg))
            ai += [self._acc_id.setdefault(a, len(self._acc_id)) for a in accs.get(m, {})]
            ao.append(len(ai))
        self.close()
        n_slots = max(len(self._slot), 1)
        from .engine import K2History
        self.k2 = K2History(self.engine, mo, mg, ao, ai, n_slots)
        self._k2_reg, self._k2_hgs = (models, {m: tuple(accs.get(m, {})) for m in hgs}, n_slots), hgs
        rows = []
        for key, vals in old.items():
            m, a, b = key.rsplit("|", 2)
            rows.append((hgs.index(m), self._acc_id[a], BUCKETS.index(b), len(vals), vals + [0.0] * (10 - len(vals))))
        if rows:
            self.k2.import_({"hg": [r[0] for r in rows], "acc": [r[1] for r in rows], "bucket": [r[2] for r in rows],
                             "count": [r[3] for r in rows], "values": [r[4] for r in rows]})

    def _k2_device(self, inputs, pos_of_all, n_out):
        """wva_k2_resolve over the batch: rep_k2 in the wva_saturation_v2 layout, and the per-slot last data replica"""
        self._k2_registry(inputs)
        cols = {k: [] for k in ("rep_total_kv_tokens", "rep_tokens_in_use", "rep_queue_length", "rep_avg_input_tokens",
                                "rep_avg_output_tokens", "rep_accelerator", "rep_slot", "rep_out_pos")}
        off, qthr, kvthr, rows = [0], [], [], []
        S = self._k2_reg[2]
        sB, sS = [0] * S, [0] * S
        for inp, pos_of in zip(inputs, pos_of_all):
            ns, model, c = inp.get("Namespace", ""), inp.get("ModelID", ""), inp["Config"]
            for i, rm in enumerate(inp.get("ReplicaMetrics", []) or []):
                s = self._slot[(ns, model, rm["VariantName"])]
                cols["rep_total_kv_tokens"].append(int(rm.get("TotalKvCapacityTokens", 0)))
                cols["rep_tokens_in_use"].append(int(rm.get("TokensInUse", 0)))
                cols["rep_queue_length"].append(int(rm.get("QueueLength", 0)))
                cols["rep_avg_input_tokens"].append(float(rm.get("AvgInputTokens", 0.0)))
                cols["rep_avg_output_tokens"].append(float(rm.get("AvgOutputTokens", 0.0)))
                cols["rep_accelerator"].append(self._acc_id[rm.get("AcceleratorName", "")])
                cols["rep_slot"].append(s)
                cols["rep_out_pos"].append(pos_of.get(i, -1))
                rec = self.store.get(ns, model, rm["VariantName"])        # params as of the start of the cycle
                p = (rec.get("VLLMParams") if rec else None) or {}
                sB[s], sS[s] = int(p.get("EffectiveMaxBatchedTokens", 0)), int(p.get("MaxNumSeqs", 0))
            off.append(len(cols["rep_slot"]))
            qthr.append(float(c.get("QueueLengthThreshold", 0.0))); kvthr.append(float(c.get("KvCacheThreshold", 0.0)))
        return self.k2.resolve(dict(cols, model_replica_off=off, n_out=n_out, slot_max_batched_tokens=sB,
                                    slot_max_num_seqs=sS, cfg_queue_threshold=qthr, cfg_kv_threshold=kvthr)), off

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

    # -- the host step around the analysis: store updates, then the zero-replica fallbacks ---------------------------
    def store_update(self, ns, model, variant, accelerator, gpu_count, num_gpu_blocks, block_size, total_kv_tokens, effective):
        """a live capacity into the store (analyzer.go:184-196), the record's VLLMParams kept"""
        old = self.store.get(ns, model, variant)
        self.store.update(ns, model, variant, {"AcceleratorName": accelerator, "GpuCount": gpu_count, "NumGpuBlocks": num_gpu_blocks,
                                               "BlockSize": block_size, "TotalKvCapacityTokens": total_kv_tokens,
                                               "EffectiveCapacity": effective, "VLLMParams": old.get("VLLMParams") if old else None,
                                               "LearnedFrom": "live"})

    def fallback_capacity(self, ns, model, variant, accelerator, gpu_count, kv_thr, avg_in, avg_out) -> float:
        """the per-replica capacity of a variant without a replica with capacity data (:317-324), read from the store
        after this cycle's updates; 0.0 = none"""
        fb, rec = 0.0, self.store.get(ns, model, variant)
        if rec is not None and rec.get("EffectiveCapacity", 0) > 0:
            fb = self._stored_capacity(rec, model, kv_thr, avg_in, avg_out)
        elif rec is not None and rec.get("VLLMParams"):
            c2 = self.store.find_compatible(model, accelerator, gpu_count, rec["VLLMParams"])
            if c2 is not None:
                fb = float(c2.get("EffectiveCapacity", 0))
        return fb

    # -- Analyze ------------------------------------------------------------------------------------------------------
    def analyze(self, inp: dict) -> dict:
        """AnalyzerInput {ModelID, Namespace, ReplicaMetrics, VariantStates, Config, SchedulerQueue} -> AnalyzerResult."""
        return self.analyze_batch([inp])[0]

    def analyze_batch(self, inputs):
        mvo, vro = [0], [0]
        rep = {k: [] for k in ("tk", "tu", "ql", "ai", "ao", "hr", "k2")}
        order, vcur, vpen, vfb, cfg = [], [], [], [], ([], [], [])
        qs, qb, any_queue = [], [], False
        meta, pos_all = [], []
        for inp in inputs:
            model, ns, c = inp.get("ModelID", ""), inp.get("Namespace", ""), inp["Config"]
            rms, states = inp.get("ReplicaMetrics", []) or [], inp.get("VariantStates", []) or []
            gpus = {s["VariantName"]: int(s.get("GPUsPerReplica", 0)) for s in states}
            kv_thr = float(c.get("KvCacheThreshold", 0.0))
            # phase 1 in slice order: the k2 chain mutates the history, the store is updated with live data
            k2_of, eff_of = {}, {}
            for i, rm in enumerate(rms):
                if self.device_history or int(rm.get("TotalKvCapacityTokens", 0)) <= 0:
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
            pos_all.append(pos_of)
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
        if self.device_history:
            k2out, k2off = self._k2_device(inputs, pos_all, len(rep["tk"]))
            d["rep_k2"] = k2out["out_rep_k2"]
        out = self.engine.saturation_v2(d)
        # the live capacities go into the store (analyzer.go:184-196, VLLMParams preserved) ...
        for mi, (inp, names, by_var, accel, cost, gpus, avg_of) in enumerate(meta):
            rms = inp.get("ReplicaMetrics", []) or []
            ns, model = inp.get("Namespace", ""), inp.get("ModelID", "")

            def update(v, i, eff):
                self.store_update(ns, model, v, rms[i].get("AcceleratorName", ""), gpus.get(v, 0), int(rms[i].get("NumGpuBlocks", 0)),
                                  int(rms[i].get("BlockSize", 0)), int(rms[i]["TotalKvCapacityTokens"]), eff)
            for k, v in enumerate(names):
                vi = mvo[mi] + k
                if self.device_history:                     # once per slot: its last data replica of the cycle
                    s = self._slot[(ns, model, v)]
                    last = int(k2out["slot_last_rep"][s])
                    if last >= 0:
                        update(v, last - k2off[mi], int(k2out["slot_effective"][s]))
                    continue
                for j, i in enumerate(by_var.get(v, [])):
                    if int(rms[i].get("TotalKvCapacityTokens", 0)) > 0:
                        update(v, i, int(out["rep_effective"][vro[vi] + j]))
        # ... before the variants without ready replicas look a capacity up (:317-324); those models are evaluated again
        any_fb = False
        for mi, (inp, names, by_var, accel, cost, gpus, avg_of) in enumerate(meta):
            rms, states = inp.get("ReplicaMetrics", []) or [], inp.get("VariantStates", []) or []
            ns, model, kv_thr = inp.get("Namespace", ""), inp.get("ModelID", ""), cfg[0][mi]
            for k, st_ in enumerate(states):
                v = st_["VariantName"]
                if any(int(rms[i].get("TotalKvCapacityTokens", 0)) > 0 for i in by_var.get(v, [])):
                    continue
                fb = self.fallback_capacity(ns, model, v, accel.get(v, ""), int(st_.get("GPUsPerReplica", 0)), kv_thr, avg_of[0], avg_of[1])
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
                vc = vc_of.get(n, {})
                decisions.append(_v2_decision(r.get("ModelID", ""), r.get("Namespace", ""), n, vc.get("AcceleratorName", ""),
                                              float(vc.get("Cost", 0.0)), int(st.get(n, {}).get("CurrentReplicas", 0)),
                                              int(tgt[mvo[mi] + k]), r["Result"], self.name()))
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


# ======================================================================================================================
# the V2 engine's cycle (optimizeV2, engines/saturation/engine.go:397-488)
# ======================================================================================================================
def _v2_decision(model, ns, name, acc, cost, current, target, result, optimizer_name):
    """CostAwareOptimizer's decision for one variant (cost_aware_optimizer.go), as CostAwareOptimizer.optimize makes it"""
    if target > current:
        action, reason = "scale-up", "V2 scale-up (optimizer: %s, required: %.0f)" % (optimizer_name, result.get("RequiredCapacity", 0.0))
    elif target < current:
        action, reason = "scale-down", "V2 scale-down (optimizer: %s, spare: %.0f)" % (optimizer_name, result.get("SpareCapacity", 0.0))
    else:
        action, reason = "no-change", "V2 steady state"
    return {"VariantName": name, "ModelID": model, "Namespace": ns, "AcceleratorName": acc, "Cost": cost,
            "CurrentReplicas": current, "TargetReplicas": target, "Action": action, "Reason": reason}


def _apply_enforced(d, enforced, optimizer_name):
    """applyEnforcedTargetsToDecisions (engine_v2.go:106-127) for one decision"""
    if enforced != d["TargetReplicas"]:
        d["TargetReplicas"] = enforced
        c = d["CurrentReplicas"]
        d["Action"] = "scale-up" if enforced > c else ("scale-down" if enforced < c else "no-change")
        d["Reason"] = "V2 %s (optimizer: %s, enforced)" % (d["Action"], optimizer_name)


def optimize_v2(analyzer, optimizer, enforcer, inputs, scale_to_zero=None):
    """optimizeV2 on the host: AnalyzerInputs of the models that make a request -> analyze_batch -> Optimize ->
    EnforcePolicy per model (extractTargetsFromDecisions / buildVariantAnalysesFromDecisions) -> the enforced targets
    applied to the decisions.  scale_to_zero: per input, ScaleToZero enabled (default off)."""
    results = analyzer.analyze_batch(inputs)
    reqs = [{"ModelID": i.get("ModelID", ""), "Namespace": i.get("Namespace", ""), "Result": r, "VariantStates": i.get("VariantStates", [])}
            for i, r in zip(inputs, results)]
    decisions = optimizer.optimize(reqs)
    of = {}
    for d in decisions:
        of.setdefault((d["ModelID"], d["Namespace"]), []).append(d)
    for k, req in enumerate(reqs):
        mine = of.get((req["ModelID"], req["Namespace"]), [])
        targets = {d["VariantName"]: d["TargetReplicas"] for d in mine}
        analyses = [{"VariantName": d["VariantName"], "AcceleratorName": d["AcceleratorName"], "Cost": d["Cost"],
                     "ReplicaCount": d["CurrentReplicas"]} for d in mine]
        enforced, _ = enforcer.enforce_policy(req["ModelID"], req["Namespace"], targets, analyses,
                                              bool(scale_to_zero[k]) if scale_to_zero is not None else False)
        for d in mine:
            if d["VariantName"] in enforced:
                _apply_enforced(d, enforced[d["VariantName"]], optimizer.name())
    return decisions


def ingest_v2_decisions(ing, analyzer, models, variant_names, accelerator_names, gpus_per_replica, optimizer_name="cost-aware"):
    """One V2 cycle through an `IngestV2` whose columns the collector has written: analyze() -> the host step on
    `analyzer`'s capacity store (SaturationAnalyzerV2.store_update once per store slot, then fallback_capacity for the
    variants without a replica with capacity data: the same code analyze_batch runs) -> decide() -> the VariantDecision
    dicts optimize_v2 returns, in registry order.  models: [(ModelID, Namespace)] per registry model; variant_names /
    accelerator_names / gpus_per_replica: per registry variant."""
    r, c = ing.analyze(), ing.cols
    mvo = ing.model_variant_off
    model_of = np.repeat(np.arange(len(mvo) - 1), np.diff(mvo))
    vslot = ing.var_store_slot
    last = r["slot_last_rep"][vslot] if len(vslot) else np.zeros(0, np.int32)
    for v in np.flatnonzero(last >= 0):                    # once per store slot: its last data replica of the cycle
        v, rep = int(v), int(last[v])
        pod, (model, ns) = int(r["rep_pod"][rep]), models[model_of[v]]
        analyzer.store_update(ns, model, variant_names[v], accelerator_names[v], int(gpus_per_replica[v]),
                              int(c["num_gpu_blocks"][pod]), int(c["block_size"][pod]), int(r["rep_total_kv_tokens"][rep]),
                              int(r["slot_effective"][vslot[v]]))
    fb = c["var_fallback_capacity"]
    fb[:] = 0.0
    has_req = r["mod_has_request"]
    for v in np.flatnonzero(r["var_no_data"]):
        v = int(v)
        m = int(model_of[v])
        if not has_req[m]:
            continue
        model, ns = models[m]
        fb[v] = analyzer.fallback_capacity(ns, model, variant_names[v], accelerator_names[v] if r["variant_replica_off"][v + 1] > r["variant_replica_off"][v] else "",
                                           int(gpus_per_replica[v]), float(c["cfg_kv_threshold"][m]),
                                           float(r["mod_avg_input_tokens"][m]), float(r["mod_avg_output_tokens"][m]))
    r = ing.decide()
    vro = r["variant_replica_off"]
    out = []
    for m in np.flatnonzero(has_req):
        m = int(m)
        model, ns = models[m]
        res = {"RequiredCapacity": float(r["mod_required_capacity"][m]), "SpareCapacity": float(r["mod_spare_capacity"][m])}
        for v in range(int(mvo[m]), int(mvo[m + 1])):
            rep = vro[v + 1] > vro[v]
            d = _v2_decision(model, ns, variant_names[v], accelerator_names[v] if rep else "", float(c["var_cost"][v]) if rep else 0.0,
                             int(c["var_current"][v]), int(r["var_optimizer_target"][v]), res, optimizer_name)
            _apply_enforced(d, int(r["var_target"][v]), optimizer_name)
            out.append(d)
    return out
