"""The V2 cycle from metric batch to decisions through wva_ingest_v2 (analyze -> host store step -> decide), against a
reference composed without the device:

    tests/collector_v2_ref.collect -> SaturationAnalyzerV2's host k2 chain + store step -> oracle.saturation_v2
    -> oracle.cost_aware_optimize -> oracle.enforce (pipeline.optimize_v2), with the history held to tests/k2_oracle

CPU: struct images, the V2 fold rules of the restated collector, fixture coverage.  GPU: bit-equal decisions, store
records and k2 history with one history carried across the cycles (20 cycles at 1 and 1 000 models, 3 at 10 000: the
Python reference takes about 30 s a cycle there); registry rejection; an empty registry; the V1 ingest graph beside a live
V2 one."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import collector_v2_ref as cv
from tests.k2_oracle import K2Oracle
from tests.test_pipeline_v2 import OracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_struct_images_match_header(pkg):
    code = r'''
#include <stdio.h>
#include "wva_b200.h"
int main(){printf("%zu %zu\n", sizeof(wva_ingest_v2_columns), sizeof(wva_ingest_v2_results));return 0;}
'''
    with tempfile.TemporaryDirectory() as td:
        open(os.path.join(td, "s.c"), "w").write(code)
        subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(td, "s"), os.path.join(td, "s.c")],
                       check=True)
        out = subprocess.run([os.path.join(td, "s")], capture_output=True, text=True, check=True).stdout.split()
    abi = pkg._abi
    assert [C.sizeof(abi.IngestV2Columns), C.sizeof(abi.IngestV2Results)] == [int(x) for x in out]
    assert [f for f, _ in abi.IngestV2Columns._fields_[4:]] == [k for k, _, _ in abi.INGEST_V2_COLUMNS]
    assert [f for f, _ in abi.IngestV2Results._fields_] == [k for k, _, _ in abi.INGEST_V2_RESULTS]


def _one(vec, **kw):
    v = {k: [] for k in cv.VECTORS}
    v.update(vec)
    recs = cv.collect(v, {"p1": "va", "p2": "va", "p3": "vb"}, {"va": "H100", "vb": "A100"}, {"va": 1.0, "vb": 2.0},
                      {"va": 0, "vb": 1})
    return {r["PodName"]: r for r in recs}


def test_collector_v2_fold_rules():
    p1, p2 = {"pod": "p1"}, {"pod_name": "p2"}
    cc = lambda lab, b, s: ({**lab, "num_gpu_blocks": b, "block_size": s}, 1.0)
    # duplicates: the later sample wins
    r = _one({"kv": [(p1, 0.2), (p1, 0.5)], "queue": [(p1, 3.0), (p1, 4.9)]})
    assert r["p1"]["KvCacheUsage"] == 0.5 and r["p1"]["QueueLength"] == 4
    # NaN / Inf avg_* do not overwrite; a hit rate outside [0, 1] or non-finite does not either
    r = _one({"kv": [(p1, 0.1)], "avg_output": [(p1, 120.0), (p1, float("nan")), (p1, float("inf"))],
              "avg_input": [(p1, -float("inf")), (p1, 7.0), (p1, float("nan"))],
              "hit_rate": [(p1, 0.25), (p1, 1.5), (p1, -0.1), (p1, float("nan"))]})
    assert (r["p1"]["AvgOutputTokens"], r["p1"]["AvgInputTokens"], r["p1"]["PrefixCacheHitRate"]) == (120.0, 7.0, 0.25)
    # missing or zero cache config: no capacity data
    r = _one({"kv": [(p1, 0.5), (p2, 0.5)], "cache_config": [cc(p2, "0", "16")]})
    assert r["p1"]["TotalKvCapacityTokens"] == 0 and r["p2"]["TotalKvCapacityTokens"] == 0 and r["p2"]["TokensInUse"] == 0
    # hasCacheConfig stays set once both were > 0; an absent / unparsable label keeps the value
    r = _one({"kv": [(p1, 0.5)], "cache_config": [cc(p1, "100", "16"), cc(p1, "", "x"), cc(p1, "200", "")]})
    assert r["p1"]["TotalKvCapacityTokens"] == 3200 and r["p1"]["TokensInUse"] == 1600
    # blocks * size overflow saturates at INT64_MAX
    r = _one({"kv": [(p1, 1.0)], "cache_config": [cc(p1, str(1 << 40), str(1 << 30))]})
    assert r["p1"]["TotalKvCapacityTokens"] == cv.INT64_MAX and r["p1"]["TokensInUse"] == cv.INT64_MIN   # int64(2^63)
    # pods with only V2 vectors are skipped; unknown pods and samples without a pod label are skipped
    r = _one({"kv": [({"pod": "zz"}, 0.5), ({}, 0.5)], "cache_config": [cc(p1, "100", "16")], "avg_output": [(p2, 5.0)]})
    assert r == {}
    # .5 ties of math.Round round away from zero
    assert [cv.go_round(x) for x in (0.5, 1.5, 2.5, -0.5, -2.5, 0.49999999999999994)] == [1.0, 2.0, 3.0, -1.0, -3.0, 0.0]
    r = _one({"kv": [(p1, 1.0 / 64.0), (p2, 3.0 / 64.0)], "queue": [(p2, 1.0)], "cache_config": [cc(p1, "2", "16"), cc(p2, "2", "16")]})
    assert r["p1"]["TokensInUse"] == 1 and r["p2"]["TokensInUse"] == 2 and r["p2"]["QueueLength"] == 1


def _coverage(fl, vec):
    reg = cv.Registry(fl)
    pods = {cv._pod(lab) for k in ("kv", "queue") for lab, _ in vec[k]}
    seen = {"dup_kv": False, "bad_avg": False, "bad_rate": False, "zero_cc": False, "overflow": False, "only_v2": False,
            "unknown": False, "tie": False, "unparsed": False}
    cnt = {}
    for lab, _ in vec["kv"]:
        cnt[cv._pod(lab)] = cnt.get(cv._pod(lab), 0) + 1
    seen["dup_kv"] = any(c > 1 for p, c in cnt.items() if p in reg.slot_of)
    seen["bad_avg"] = any(not math.isfinite(x) for k in ("avg_output", "avg_input") for _, x in vec[k])
    seen["bad_rate"] = any(math.isfinite(x) and not 0 <= x <= 1 for _, x in vec["hit_rate"])
    seen["zero_cc"] = any(lab.get("num_gpu_blocks") == "0" for lab, _ in vec["cache_config"])
    seen["unparsed"] = any(lab.get("num_gpu_blocks") == "12x" for lab, _ in vec["cache_config"])
    seen["overflow"] = any(lab.get("num_gpu_blocks") == str(1 << 40) for lab, _ in vec["cache_config"])
    seen["only_v2"] = any(cv._pod(lab) not in pods and cv._pod(lab) in reg.slot_of for lab, _ in vec["avg_output"])
    seen["unknown"] = any(cv._pod(lab) and cv._pod(lab) not in reg.slot_of for lab, _ in vec["kv"])
    seen["tie"] = any(lab.get("num_gpu_blocks") == "4096" for lab, _ in vec["cache_config"])
    return seen


def test_fixture_covers_every_fold_case():
    fl = cv.fleet(200, 8, seed=1)
    vec, state, mod = cv.cycle(fl, 2)
    seen = _coverage(fl, vec)
    assert all(seen.values()), seen
    reg = cv.Registry(fl)
    inputs, s2z, _, per = reg.reference_inputs(vec, state, mod)
    assert len(inputs) < len(fl["models"])                                       # models with no reporting pod
    assert any(x["TotalKvCapacityTokens"] == cv.INT64_MAX for i in inputs for x in i["ReplicaMetrics"])
    assert any(all(x["TotalKvCapacityTokens"] <= 0 for x in i["ReplicaMetrics"] if x["VariantName"] == s["VariantName"])
               for i in inputs for s in i["VariantStates"])                     # variants that need the store fallback
    assert any(s2z) and mod["err"].any()
    assert len({m for m, _ in fl["models"]}) < len(fl["models"])                 # modelIDs shared across namespaces


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _same(a, b):
    if isinstance(a, float) and isinstance(b, float):
        return (math.isnan(a) and math.isnan(b)) or a == b
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _k2_columns(reg, per, store):
    """the cycle's replicas as wva_k2_in columns (model group m = model m) for the k2 oracle"""
    cols = {k: [] for k in ("rep_total_kv_tokens", "rep_tokens_in_use", "rep_queue_length", "rep_avg_input_tokens",
                            "rep_avg_output_tokens", "rep_accelerator", "rep_slot")}
    off = [0]
    for m in range(len(reg.fl["models"])):
        for r in per.get(m, []):
            k = reg.variant_rank[r["VariantName"]]
            cols["rep_total_kv_tokens"].append(r["TotalKvCapacityTokens"]); cols["rep_tokens_in_use"].append(r["TokensInUse"])
            cols["rep_queue_length"].append(r["QueueLength"]); cols["rep_avg_input_tokens"].append(r["AvgInputTokens"])
            cols["rep_avg_output_tokens"].append(r["AvgOutputTokens"]); cols["rep_accelerator"].append(int(reg.var_acc[k]))
            cols["rep_slot"].append(int(reg.var_slot[k]))
        off.append(len(cols["rep_slot"]))
    B, S = reg.slot_params(store)
    return dict(cols, model_replica_off=off, slot_max_batched_tokens=B, slot_max_num_seqs=S,
                cfg_queue_threshold=[c["QueueLengthThreshold"] for c in reg.fl["cfg"]],
                cfg_kv_threshold=[c["KvCacheThreshold"] for c in reg.fl["cfg"]])


def run_parity(pkg, engine, oracle, n_models, max_variants, n_cycles, seed):
    fl = cv.fleet(n_models, max_variants, seed)
    reg = cv.Registry(fl)
    oe = OracleEngine(oracle)
    ref = pkg.SaturationAnalyzerV2(oe)                       # host k2 chain, oracle analysis
    dev = pkg.SaturationAnalyzerV2(engine)                   # the store the device path's host step works on
    reg.seed_store(ref.store); reg.seed_store(dev.store)
    orc = K2Oracle(*reg.k2_registry())
    stats = {"decisions": 0, "fallback": 0, "enforced": 0, "changed_cols": 0, "deployment_estimate": 0, "compatible": 0}
    stored, find = dev._stored_capacity, dev.store.find_compatible

    def stored_counted(rec, *a):                             # estimateStoredCapacity's deployment branch (:365-415)
        if rec.get("LearnedFrom") != "live" and rec.get("VLLMParams") and a[3] > 0:
            stats["deployment_estimate"] += 1
        return stored(rec, *a)

    def find_counted(*a):
        c = find(*a)
        stats["compatible"] += c is not None
        return c
    dev._stored_capacity, dev.store.find_compatible = stored_counted, find_counted
    with pkg.K2History(engine, *reg.k2_registry()) as h, \
            pkg.IngestV2(engine, reg.mvo, reg.vso, reg.var_acc, reg.var_slot, h) as ing:
        prev = None
        for c in range(n_cycles):
            vec, state, mod = cv.cycle(fl, seed * 1000 + c)
            inputs, s2z, count, per = reg.reference_inputs(vec, state, mod)
            assert orc.resolve(_k2_columns(reg, per, ref.store)) is not None
            want = pkg.optimize_v2(ref, pkg.CostAwareOptimizer(oe), pkg.Enforcer(oe, count), inputs, s2z) if inputs else []
            reg.write(ing, pkg._abi, vec, state, mod, dev.store)
            snap = {k: v.copy() for k, v in ing.cols.items()}
            if prev is not None:
                stats["changed_cols"] += sum(not np.array_equal(snap[k], prev[k]) for k in snap)
            prev = snap
            got = pkg.ingest_v2_decisions(ing, dev, *reg.decisions_args())
            assert _same(got, want), c
            for m in range(len(fl["models"])):                # computeModelWorkloadAverages (analyzer.go:438-455)
                ai = ao = 0.0
                n = 0
                for r in per.get(m, []):
                    if r["AvgInputTokens"] > 0 or r["AvgOutputTokens"] > 0:
                        ai += r["AvgInputTokens"]; ao += r["AvgOutputTokens"]; n += 1
                if n:
                    ai /= float(n); ao /= float(n)
                got_avg = (ing.res["mod_avg_input_tokens"][m], ing.res["mod_avg_output_tokens"][m])
                assert np.array([ai, ao]).view(np.int64).tolist() == np.array(got_avg).view(np.int64).tolist(), (c, m)
            assert list(dev.store.records.items()) == list(ref.store.records.items()), c
            stats["decisions"] += len(got)
            stats["fallback"] += int((ing.cols["var_fallback_capacity"] > 0).sum())
            stats["enforced"] += sum("enforced" in d["Reason"] for d in got)
        e = h.export()
        cnt, vals = orc.export()
        assert np.array_equal(e["count"], cnt)
        assert np.array_equal(e["values"].view(np.int64), np.asarray(vals, np.float64).view(np.int64))
        assert ref.history_state() == {"%s|%s|%s" % (reg.hgs[int(e["hg"][k])], cv.ACCS[int(e["acc"][k])],
                                                    ("short", "medium", "long")[int(e["bucket"][k])]):
                                       [float(x) for x in e["values"][k, :int(e["count"][k])]]
                                       for k in range(len(e["hg"])) if e["count"][k] > 0}
    orc.close()
    return stats


@pytest.mark.gpu
@pytest.mark.parametrize("n_models,max_variants,n_cycles", [(1, 32, 20), (1000, 32, 20), (10000, 32, 3)])
def test_ingest_v2_matches_reference(pkg, engine, oracle, n_models, max_variants, n_cycles):
    s = run_parity(pkg, engine, oracle, n_models, max_variants, n_cycles, seed=n_models)
    assert s["decisions"] > 0 and s["changed_cols"] > 0
    if n_models > 1:
        assert s["fallback"] > 0 and s["enforced"] > 0 and s["deployment_estimate"] > 0 and s["compatible"] > 0, s


@pytest.mark.gpu
def test_rejected_registry_and_cycle_leave_history_unchanged(pkg, engine, oracle):
    fl = cv.fleet(50, 6, seed=3)
    reg = cv.Registry(fl)
    an = pkg.SaturationAnalyzerV2(engine)
    reg.seed_store(an.store)
    with pkg.K2History(engine, *reg.k2_registry()) as h:
        with pkg.IngestV2(engine, reg.mvo, reg.vso, reg.var_acc, reg.var_slot, h) as ing:
            vec, state, mod = cv.cycle(fl, 1)
            reg.write(ing, pkg._abi, vec, state, mod, an.store)
            pkg.ingest_v2_decisions(ing, an, *reg.decisions_args())
        before = h.export()
        bad_acc = reg.var_acc.copy()
        bad_acc[0] = 99                                                   # not registered for its history group
        bad_slot = reg.var_slot.copy()
        bad_slot[-1] = reg.n_store_slots                                  # out of range
        for acc, sl in ((bad_acc, reg.var_slot), (reg.var_acc, bad_slot)):
            with pytest.raises(pkg.WvaError):
                pkg.IngestV2(engine, reg.mvo, reg.vso, acc, sl, h)
        with pkg.IngestV2(engine, reg.mvo, reg.vso, reg.var_acc, reg.var_slot, h) as ing:
            with pytest.raises(pkg.WvaError):
                ing.decide()                                              # no analysis in this cycle
            with pytest.raises(pkg.WvaError):
                ing.write(pkg._abi.VEC_AVG_INPUT_TOKENS, [len(reg.slot_of)], [1.0])   # slot out of range
        after = h.export()
        assert np.array_equal(before["count"], after["count"])
        assert np.array_equal(before["values"].view(np.int64), after["values"].view(np.int64))


@pytest.mark.gpu
def test_empty_registry(pkg, engine):
    with pkg.K2History(engine, [0], [], [0], [], 1) as h, pkg.IngestV2(engine, [0], [0], [], [], h) as ing:
        an = pkg.SaturationAnalyzerV2(engine)
        for _ in range(2):
            ing.begin()
            assert pkg.ingest_v2_decisions(ing, an, [], [], [], []) == []


@pytest.mark.gpu
def test_v1_ingest_unchanged_beside_ingest_v2(pkg, engine):
    from tests import collector_ref as cr
    from tests.test_ingest import _registry, _vector_to_slots
    fx = cr.fixture(300, 8, seed=4)
    mvo, vso, slot_of, _ = _registry(fx)
    M, V = len(mvo) - 1, len(vso) - 1
    g = np.random.default_rng(4)

    def cycle(ing):
        ing.begin()
        ing.write(pkg._abi.VEC_KV_CACHE_USAGE, *_vector_to_slots(fx["kv"], slot_of))
        ing.write(pkg._abi.VEC_QUEUE_LENGTH, *_vector_to_slots(fx["queue"], slot_of))
        for k, v in state.items():
            ing.cols[k][:] = v
        if ing.dcols is not None:
            for k, v in dstate.items():
                ing.dcols[k][:] = v
        ing.commit()
        out = {k: v.copy() for k, v in ing.res.items()}
        if ing.dres is not None:
            out.update({"d_" + k: v.copy() for k, v in ing.dres.items()})
        return out
    state = {"var_cost": g.uniform(1, 10, V), "var_current": g.integers(0, 5, V).astype(np.int32),
             "var_desired": g.integers(0, 5, V).astype(np.int32), "var_pending": np.zeros(V, np.int32),
             "cfg_kv_threshold": np.full(M, 0.8), "cfg_queue_threshold": np.full(M, 5.0), "cfg_kv_trigger": np.full(M, 0.1),
             "cfg_queue_trigger": np.full(M, 3.0)}
    dstate = {"var_accelerator_type": (np.arange(V) % 4).astype(np.int32), "var_gpus_per_replica": np.ones(V, np.int32),
              "mod_scale_to_zero_enabled": (g.random(M) < 0.3).astype(np.uint8), "mod_request_count": np.zeros(M),
              "mod_request_error": np.zeros(M, np.uint8), "type_limit": np.full(4, 50, np.int32), "enable_limiter": np.ones(1, np.int32)}
    plain, dec = pkg.Ingest(engine, mvo, vso), pkg.Ingest(engine, mvo, vso, n_types=4)
    try:
        a0, b0 = cycle(plain), cycle(dec)
        fl = cv.fleet(100, 8, seed=9)
        reg = cv.Registry(fl)
        an = pkg.SaturationAnalyzerV2(engine)
        reg.seed_store(an.store)
        with pkg.K2History(engine, *reg.k2_registry()) as h, pkg.IngestV2(engine, reg.mvo, reg.vso, reg.var_acc, reg.var_slot, h) as ing:
            vec, st, mod = cv.cycle(fl, 5)
            reg.write(ing, pkg._abi, vec, st, mod, an.store)
            pkg.ingest_v2_decisions(ing, an, *reg.decisions_args())
            a1, b1 = cycle(plain), cycle(dec)
            for x, y in ((a0, a1), (b0, b1)):
                assert x.keys() == y.keys() and all(np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)) for k in x)
    finally:
        plain.close(); dec.close()
