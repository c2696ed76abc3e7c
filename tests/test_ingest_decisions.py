"""Decision mode of the ingest graph (wva_ingest_create_decisions): metric batch -> the cycle's final VariantDecisions
in one CUDA graph launch, against the reference composed in this file from the oracle:

    oracle.saturation_v1 -> oracle.enforce -> convertSaturationTargetsToDecisions restated below -> oracle.limit

on tests/collector_ref.py fixtures.  The GPU-count limiter's fixed-size sort is also held to oracle.limit through
wva_limit with more than 256 accelerator types."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import collector_ref as cr
from tests.test_ingest import _registry, _vector_to_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- fixtures -------------------------------------------------------------------------------------------------------
def make_case(n_models, vpm, seed, T):
    """A deployment and one cycle of metric vectors (collector_ref.fixture) with, besides what the join copes with:
    models none of whose pods report, variants without a reporting pod, KV samples on a 1/8 grid (ties in spare
    capacity), costs from a small set (ties in cost), models with every replica gone (all targets 0: the enforcer keeps
    one replica on the cheapest variant, ties broken by name), models in transition."""
    fx = cr.fixture(n_models, vpm, seed=seed)
    g = np.random.default_rng(seed + 1000)
    n_silent = max(1, n_models // 20) if n_models > 1 else 0
    silent = set(int(m) for m in g.choice(n_models, n_silent, replace=False)) if n_silent else set()
    silent_pods = {p for m in silent for va in fx["variants"][fx["models"][m]] for p in fx["pods"][va]}
    kv = []
    for i, (lab, v) in enumerate(fx["kv"]):
        if cr._pod(lab) in silent_pods:
            continue
        kv.append((lab, float(np.round(v * 8.0) / 8.0) if i % 2 == 0 else v))
    fx["kv"] = kv
    fx["queue"] = [(lab, v) for lab, v in fx["queue"] if cr._pod(lab) not in silent_pods]
    mvo, vso, slot_of, var_names = _registry(fx)
    M, V = len(mvo) - 1, len(vso) - 1
    recs = cr.collect(fx["kv"], fx["queue"], fx["pod_to_variant"])
    vidx = {n: i for i, n in enumerate(var_names)}
    cnt = np.zeros(V, np.int64)
    for r in recs:
        cnt[vidx[r["VariantName"]]] += 1
    vro = np.zeros(V + 1, np.int64); np.cumsum(cnt, out=vro[1:])
    model_of = np.repeat(np.arange(M), np.diff(mvo))
    cost = np.array([1.0, 2.5, 10.0, 40.0, 2.5])[g.integers(0, 5, V)]
    cur = cnt.astype(np.int32)
    cur[g.random(V) < 0.08] += 1                                     # in transition: metrics != current
    gone = g.random(M) < 0.15                                        # every replica of the model gone
    cur[gone[model_of]] = 0
    cost[gone[model_of]] = 2.5                                       # ... at equal cost: the name breaks the tie
    desired = (cur + g.integers(-1, 2, V)).clip(0).astype(np.int32)
    desired[gone[model_of]] = 0                                      # no scale-down in flight: every target is 0
    state = {"var_cost": cost, "var_current": cur, "var_desired": desired, "var_pending": (g.random(V) < 0.05).astype(np.int32)}
    cfg = {"cfg_kv_threshold": np.full(M, 0.8), "cfg_queue_threshold": np.full(M, 5.0), "cfg_kv_trigger": np.full(M, 0.1),
           "cfg_queue_trigger": np.full(M, 3.0)}
    batch = {"n_models": M, "n_variants": V, "n_replicas": len(recs), "model_variant_off": mvo,
             "variant_replica_off": vro.astype(np.int32), "rep_kv": np.array([r["KvCacheUsage"] for r in recs], np.float64),
             "rep_queue": np.array([r["QueueLength"] for r in recs], np.int64), **state, **cfg}
    return {"fx": fx, "mvo": mvo, "vso": vso, "slot_of": slot_of, "var_names": var_names, "cnt": cnt, "batch": batch,
            "state": state, "cfg": cfg, "T": T, "M": M, "V": V, "silent": silent}


def decision_columns(case, seed, enable=1):
    """One cycle's decision columns: accelerator types in [-1, T), GPUsPerReplica including 0 and negative values,
    scale-to-zero with request count 0 / > 0 / a failed lookup, and per-type limits around the GPUs in use — some
    binding, some not, some types without a pool (limit 0)."""
    g = np.random.default_rng(seed)
    M, V, T = case["M"], case["V"], case["T"]
    st = case["state"]
    typ = g.integers(-1, T, V).astype(np.int32) if T > 0 else np.full(V, -1, np.int32)
    gpr = np.array([-1, 0, 1, 1, 2, 4, 8])[g.integers(0, 7, V)].astype(np.int32)
    s2z = (g.random(M) < 0.35).astype(np.uint8)
    req = np.where(g.random(M) < 0.5, 0.0, g.integers(1, 50, M).astype(np.float64))
    err = (g.random(M) < 0.1).astype(np.uint8)
    used = np.zeros(max(T, 1), np.int64)
    ok = (typ >= 0) & (case["cnt"] > 0)
    np.add.at(used, typ[ok], st["var_current"][ok].astype(np.int64) * np.maximum(gpr[ok], 1))
    lim = np.zeros(T, np.int32)
    for t in range(T):
        r = g.random()
        lim[t] = 0 if r < 0.15 else (1 << 30) if r < 0.35 else int(used[t] + g.integers(-4, 24))
    return {"var_accelerator_type": typ, "var_gpus_per_replica": gpr, "mod_scale_to_zero_enabled": s2z,
            "mod_request_count": req, "mod_request_error": err, "type_limit": lim,
            "enable_limiter": np.array([enable], np.int32)}


# ---- the reference, composed --------------------------------------------------------------------------------------
def reference_cycle(oracle, case, dc):
    """optimizeV1 (engines/saturation/engine.go:281-395) for every model of the cycle, per-variant arrays + decisions"""
    b, mvo, cnt, T = case["batch"], case["mvo"], case["cnt"], case["T"]
    M, V = case["M"], case["V"]
    o = oracle.saturation_v1(b)                                      # RunSaturationAnalysis (:315)
    model_of = np.repeat(np.arange(M), np.diff(mvo))
    va = cnt > 0                                                     # a VariantSaturationAnalysis exists (analyzer.go:148-149)
    reporting = np.bincount(model_of, weights=cnt, minlength=M) > 0  # prepareModelData: no metrics -> nil (:737-742)
    tgt, app = oracle.enforce(dict(model_variant_off=mvo, mod_scale_to_zero_enabled=dc["mod_scale_to_zero_enabled"],
                                   mod_request_count=dc["mod_request_count"], mod_request_error=dc["mod_request_error"],
                                   var_cost=b["var_cost"], var_has_cost=va.astype(np.uint8), var_target=o["var_target"]))
    app = app.astype(bool) & reporting                               # the enforcer runs only on an analysis (:323-343)
    # convertSaturationTargetsToDecisions (engine.go:589-661): one decision per entry of the targets map
    decisions = []
    for v in range(V):
        m = int(model_of[v])
        if not reporting[m] or tgt[v] < 0:
            continue
        t, c = int(tgt[v]), int(b["var_current"][v])
        action = "scale-up" if t > c else "scale-down" if t < c else "no-change"   # :614-622
        g = int(dc["var_gpus_per_replica"][v])
        d = {"_v": v, "VariantName": case["var_names"][v], "ModelID": case["fx"]["models"][m], "Namespace": "ns",
             "CurrentReplicas": c, "TargetReplicas": t, "OriginalTargetReplicas": t,
             "DesiredReplicas": int(b["var_desired"][v]), "Action": action, "Reason": "saturation-only mode: " + action,
             "GPUsPerReplica": g if g > 0 else 1,                                    # :624-628
             "AcceleratorName": "", "Cost": 0.0, "SpareCapacity": 0.0,               # va == nil (:653-656)
             "GPUsAllocated": 0, "WasLimited": False, "LimitedBy": "", "DecisionSteps": []}
        if va[v]:                                                                    # :647-652
            d["AcceleratorName"] = "type-%03d" % dc["var_accelerator_type"][v] if dc["var_accelerator_type"][v] >= 0 else ""
            d["Cost"] = float(b["var_cost"][v])
            d["SpareCapacity"] = float(o["var_avg_spare_kv"][v])
        decisions.append(d)
    if dc["enable_limiter"][0] and decisions:                                        # :370
        acc = [int(dc["var_accelerator_type"][d["_v"]]) if d["AcceleratorName"] else -1 for d in decisions]
        lo = oracle.limit({"n_types": T, "acc_type": acc, "current": [d["CurrentReplicas"] for d in decisions],
                           "target": [d["TargetReplicas"] for d in decisions],
                           "gpus_per_replica": [d["GPUsPerReplica"] for d in decisions],
                           "spare": [d["SpareCapacity"] for d in decisions], "cost": [d["Cost"] for d in decisions],
                           "type_limit": dc["type_limit"]})
        for i, d in enumerate(decisions):                                            # default_limiter.go:85-97
            d["TargetReplicas"], d["GPUsAllocated"] = int(lo["target"][i]), int(lo["gpus_allocated"][i])
            d["WasLimited"] = bool(lo["was_limited"][i])
            if d["WasLimited"]:
                d["LimitedBy"] = "gpu-limiter"
            ch = d["TargetReplicas"] - d["CurrentReplicas"]
            reason = ("no scale-up (target=%d, current=%d)" % (d["TargetReplicas"], d["CurrentReplicas"]) if ch <= 0 else
                      "limited: allocated %d GPUs for +%d replicas" % (d["GPUsAllocated"], ch) if d["WasLimited"] else
                      "allocated %d GPUs for +%d replicas" % (d["GPUsAllocated"], ch))
            d["DecisionSteps"].append({"Name": "gpu-limiter", "Action": d["Action"], "TargetReplicas": d["TargetReplicas"],
                                       "Reason": reason, "WasConstrained": d["WasLimited"]})
    exp = {"has_decision": np.zeros(V, np.uint8), "original_target": np.full(V, -1, np.int32), "target": np.full(V, -1, np.int32),
           "gpus_allocated": np.zeros(V, np.int32), "was_limited": np.zeros(V, np.uint8), "action": np.zeros(V, np.int8),
           "mod_enforcer_applied": app.astype(np.uint8)}
    sign = {"scale-up": 1, "scale-down": -1, "no-change": 0}
    for d in decisions:
        v = d["_v"]
        exp["has_decision"][v] = 1
        exp["original_target"][v], exp["target"][v] = d["OriginalTargetReplicas"], d["TargetReplicas"]
        exp["gpus_allocated"][v], exp["was_limited"][v] = d["GPUsAllocated"], d["WasLimited"]
        exp["action"][v] = sign[d["Action"]]
    return o, exp, decisions


def coverage(case, dc, o, exp, decisions):
    """which of the situations the decision stage must reproduce occur in this cycle"""
    cnt, M, T = case["cnt"], case["M"], case["T"]
    mvo = case["mvo"]
    model_of = np.repeat(np.arange(M), np.diff(mvo))
    va = cnt > 0
    has = exp["has_decision"].astype(bool)
    cur = case["state"]["var_current"]
    cand = has & (exp["original_target"] > cur)
    typ, lim = dc["var_accelerator_type"], dc["type_limit"]
    t_ok = (typ >= 0) & va
    s2z = dc["mod_scale_to_zero_enabled"].astype(bool)
    app = exp["mod_enforcer_applied"].astype(bool)
    rep = np.bincount(model_of, weights=cnt, minlength=M) > 0
    def ties(x):
        return x.size != np.unique(x).size
    c = {"transition": bool((has & (cur != cnt)).any()), "silent model": bool((~rep).any() and rep.any()),
         # (CalculateSaturationTargets only maps variants that have an analysis, so the `va == nil` decision branch is
         # not reachable from a cycle's metrics; the variants are there, without a decision)
         "no-pod variant in a reporting model": bool((~va & rep[model_of]).any()),
         "s2z, count 0": bool((s2z & app).any()),
         "s2z, count > 0": bool((s2z & rep & ~app & (dc["mod_request_count"] > 0) & (dc["mod_request_error"] == 0)).any()),
         "s2z, lookup error": bool((s2z & rep & (dc["mod_request_error"] != 0)).any()),
         "keep one on the cheapest": bool((~s2z & app).any()),
         "GPUsPerReplica 0": bool((has & (dc["var_gpus_per_replica"] == 0)).any()),
         "type -1": bool((has & va & (typ < 0)).any())}
    if dc["enable_limiter"][0] and T > 0:
        c["type without a pool"] = bool((cand & t_ok & (lim[np.clip(typ, 0, None)] == 0)).any())
        c["binding limit"] = bool((cand & t_ok & (exp["was_limited"] != 0) & (lim[np.clip(typ, 0, None)] > 0)).any())
        c["non-binding limit"] = bool((cand & t_ok & (exp["was_limited"] == 0)).any())
        c["spare ties"] = ties(o["var_avg_spare_kv"][cand])
        c["cost ties"] = ties(case["batch"]["var_cost"][cand & va])
    return c


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_decision_struct_images_match_header(pkg):
    """ctypes images of the ingest structs vs sizeof() from the C header (compiled with the host compiler)."""
    code = r'''
#include <stdio.h>
#include "wva_b200.h"
int main(){printf("%zu %zu %zu %zu\n", sizeof(wva_ingest_columns), sizeof(wva_ingest_results),
 sizeof(wva_ingest_decision_columns), sizeof(wva_ingest_decision_results));return 0;}
'''
    with tempfile.TemporaryDirectory() as td:
        open(os.path.join(td, "s.c"), "w").write(code)
        subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(td, "s"),
                        os.path.join(td, "s.c")], check=True)
        out = subprocess.run([os.path.join(td, "s")], capture_output=True, text=True, check=True).stdout.split()
    abi = pkg._abi
    got = [C.sizeof(x) for x in (abi.IngestColumns, abi.IngestResults, abi.IngestDecisionColumns, abi.IngestDecisionResults)]
    assert got == [int(x) for x in out]


def test_decision_fixtures_cover_every_case(oracle):
    """The parity fixtures below reach every situation the decision stage distinguishes (checked on the oracle)."""
    case = make_case(400, 32, 2, 8)
    seen = {}
    for cycle in range(3):
        dc = decision_columns(case, 500 + cycle, enable=1)
        o, exp, dec = reference_cycle(oracle, case, dc)
        for k, v in coverage(case, dc, o, exp, dec).items():
            seen[k] = seen.get(k, False) or v
    missing = [k for k, v in seen.items() if not v]
    assert not missing, missing


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _load(ing, case, dc):
    fx, slot_of = case["fx"], case["slot_of"]
    ing.begin()
    ing.write(0, *_vector_to_slots(fx["kv"], slot_of))
    ing.write(1, *_vector_to_slots(fx["queue"], slot_of))
    for k, v in {**case["state"], **case["cfg"]}.items():
        ing.cols[k][:] = v
    if ing.dcols is not None:
        for k, v in dc.items():
            ing.dcols[k][:] = v


PLAIN_KEYS = ("var_target", "var_replica_count", "var_non_saturated", "var_avg_spare_kv", "var_avg_spare_queue", "mod_flags",
              "mod_total_replicas", "partials")


def _check(ing, exp, o, what):
    for k, v in exp.items():
        assert np.array_equal(ing.dres[k], v), (k, what, np.flatnonzero(ing.dres[k] != v)[:10])
    for k in ("var_target", "var_non_saturated", "mod_flags", "mod_total_replicas", "partials"):
        assert np.array_equal(ing.res[k], o[k]), (k, what)
    for k in ("var_avg_spare_kv", "var_avg_spare_queue"):
        assert np.array_equal(ing.res[k].view(np.uint64), o[k].view(np.uint64)), (k, what)


@pytest.mark.gpu
@pytest.mark.parametrize("n_models,vpm,seed,T", [(50, 6, 1, 4), (400, 32, 2, 8), (3, 1, 3, 2), (2000, 16, 4, 0),
                                                 (1000, 32, 6, 300), (10000, 32, 5, 8)])
def test_decisions_match_reference(pkg, engine, oracle, n_models, vpm, seed, T):
    """Bit-for-bit parity of every decision result with the composed reference, over cycles of one graph that change
    the limits, request counts, scale-to-zero flags, GPUsPerReplica, types and the limiter switch between them."""
    case = make_case(n_models, vpm, seed, T)
    ing = pkg.Ingest(engine, case["mvo"], case["vso"], n_types=T)
    try:
        for cycle, enable in enumerate((1, 0, 1)):
            dc = decision_columns(case, seed * 10 + cycle, enable=enable)
            o, exp, _ = reference_cycle(oracle, case, dc)
            _load(ing, case, dc)
            ing.commit()
            assert np.array_equal(ing.res["var_replica_count"], case["cnt"]), cycle
            _check(ing, exp, o, (cycle, enable))
        # a cycle in which nothing reports: no model has an analysis, so no decision and no enforcer
        ing.begin()
        ing.commit()
        assert not ing.dres["has_decision"].any() and not ing.dres["mod_enforcer_applied"].any()
    finally:
        ing.close()


@pytest.mark.gpu
def test_decision_mode_leaves_the_plain_results_unchanged(pkg, engine, oracle):
    """var_target, the analyses and the partials of the decision mode equal the plain graph's on the same inputs."""
    case = make_case(400, 32, 7, 8)
    dc = decision_columns(case, 70)
    plain = pkg.Ingest(engine, case["mvo"], case["vso"])
    dec = pkg.Ingest(engine, case["mvo"], case["vso"], n_types=8)
    try:
        assert plain.dres is None and dec.dres is not None
        _load(plain, case, dc)
        _load(dec, case, dc)
        a, b = plain.commit(), dec.commit()
        for k in PLAIN_KEYS:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    finally:
        plain.close()
        dec.close()


@pytest.mark.gpu
def test_decision_graph_captures_without_host_sync(pkg, engine):
    """The limiter stage is enqueued inside stream capture (a host synchronisation there fails the capture, and with it
    create); empty registries and T = 0 capture too."""
    for mvo, vso, T in (([0, 2], [0, 1, 3], 300), ([0], [0], 0), ([0, 0], [0], 5), ([0, 1], [0, 2], 0)):
        ing = pkg.Ingest(engine, mvo, vso, n_types=T)
        try:
            before = engine.launch_count()
            ing.begin()
            ing.commit()
            assert engine.launch_count() > before
            assert ing.dcols["type_limit"].size == T
        finally:
            ing.close()
    with pytest.raises(pkg.WvaError):
        pkg.Ingest(engine, [0, 1], [0, 2], n_types=-2)


@pytest.mark.gpu
def test_ingest_decisions_host_twin(pkg, engine, oracle):
    """pipeline.ingest_decisions turns the device results into the reference's VariantDecision dicts."""
    case = make_case(60, 6, 11, 4)
    ing = pkg.Ingest(engine, case["mvo"], case["vso"], n_types=4)
    try:
        for cycle, enable in enumerate((1, 0)):
            dc = decision_columns(case, 110 + cycle, enable=enable)
            _, _, ref = reference_cycle(oracle, case, dc)
            _load(ing, case, dc)
            ing.commit()
            models = [(m, "ns") for m in case["fx"]["models"]]
            acc = ["type-%03d" % t if t >= 0 else "" for t in dc["var_accelerator_type"]]
            got = pkg.pipeline.ingest_decisions(ing, models, case["var_names"], acc)
            assert len(got) == len(ref) > 0
            for g, r in zip(got, ref):
                r = {k: v for k, v in r.items() if k != "_v"}
                assert g == r, (g, r)
    finally:
        ing.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_limit_past_256_types_matches_oracle(engine, oracle, seed):
    """wva_limit with T = 300: the "" segment (key T) and the types >= 256 must not alias types in the low 8 bits."""
    g = np.random.default_rng(seed)
    D, T = 6000, 300
    hot = np.array([0, 44, 45, 256, 299])                           # 300 & 255 = 44, 256 & 255 = 0, 301 & 255 = 45
    acc = np.where(g.random(D) < 0.7, hot[g.integers(0, hot.size, D)], g.integers(-1, T, D)).astype(np.int32)
    acc[g.random(D) < 0.1] = -1
    cur = g.integers(0, 6, D).astype(np.int32)
    tgt = (cur + g.integers(-2, 5, D)).clip(0).astype(np.int32)
    gpr = np.array([0, 1, 2, 4])[g.integers(0, 4, D)].astype(np.int32)
    used = np.zeros(T, np.int64)
    ok = acc >= 0
    np.add.at(used, acc[ok], cur[ok].astype(np.int64) * gpr[ok])
    lim = (used + g.integers(0, 40, T)).astype(np.int32)
    d = {"n_types": T, "acc_type": acc, "current": cur, "target": tgt, "gpus_per_replica": gpr,
         "spare": np.round(g.random(D) * 4) / 4, "cost": np.array([1.0, 2.0, 3.0])[g.integers(0, 3, D)], "type_limit": lim}
    got, ref = engine.limit(d), oracle.limit(d)
    assert ref["was_limited"].any() and (ref["gpus_allocated"] > 0).any()
    for k in ("target", "gpus_allocated", "was_limited"):
        assert np.array_equal(got[k], ref[k]), k
