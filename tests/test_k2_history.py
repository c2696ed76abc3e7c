"""The V2 analyzer's k2 priority chain (computeK2, internal/engines/analyzers/saturation_v2/analyzer.go:218-262) with its
rolling history (history.go) resolved on the device: wva_k2_resolve / engine.K2History.

CPU: the reference's own k2 cases (analyzer_test.go:88-224) through the host chain of SaturationAnalyzerV2 and through
the C++ oracle (tests/k2_oracle), and the oracle against the host chain over seeded multi-cycle sequences (rep_k2 and
the whole history after every cycle).  GPU: the device against the oracle bit for bit over 20 cycles at 1, 1 000 and
100 000 model groups (both ring placements), atomicity of rejected calls, idempotence of the analysis, export/import
resumption, and SaturationAnalyzerV2 with device history against its host history end to end.
"""
import math

import numpy as np
import pytest

from tests.k2_oracle import K2Oracle
from tests.test_pipeline_v2 import CFG, OracleEngine, inp, rm, st

BUCKETS = ("short", "medium", "long")


# ---------------------------------------------------------------------------------------------------------------------
# named cycles -> the integer registry and columns of wva_k2_resolve
# ---------------------------------------------------------------------------------------------------------------------
class Encoder:
    """name -> id maps as a caller keeps them: accelerator names ("" included), store slots namespace|model|variant, and
    one history group per modelID whose model groups are the inputs in list order."""

    def __init__(self, cycles):
        self.acc, self.slot = {}, {}
        self.models = [i["ModelID"] for i in cycles[0]]
        assert all([i["ModelID"] for i in c] == self.models for c in cycles), "one registry for the whole sequence"
        self.hgs = list(dict.fromkeys(self.models))
        accs = {m: {} for m in self.hgs}
        for c in cycles:
            for i in c:
                for r in i["ReplicaMetrics"]:
                    accs[i["ModelID"]][r.get("AcceleratorName", "")] = None
                    self.slot.setdefault((i["Namespace"], i["ModelID"], r["VariantName"]), len(self.slot))
        self.mo, self.mg, self.ao, self.ai = [0], [], [0], []
        for m in self.hgs:
            self.mg += [g for g, x in enumerate(self.models) if x == m]
            self.mo.append(len(self.mg))
            self.ai += [self.acc.setdefault(a, len(self.acc)) for a in accs[m]]
            self.ao.append(len(self.ai))
        self.n_slots = max(len(self.slot), 1)

    def registry(self):
        return self.mo, self.mg, self.ao, self.ai, self.n_slots

    def columns(self, cycle, params):
        c = {k: [] for k in ("rep_total_kv_tokens", "rep_tokens_in_use", "rep_queue_length", "rep_avg_input_tokens",
                             "rep_avg_output_tokens", "rep_accelerator", "rep_slot")}
        off, sB, sS = [0], [0] * self.n_slots, [0] * self.n_slots
        for i in cycle:
            for r in i["ReplicaMetrics"]:
                s = self.slot[(i["Namespace"], i["ModelID"], r["VariantName"])]
                c["rep_total_kv_tokens"].append(r["TotalKvCapacityTokens"]); c["rep_tokens_in_use"].append(r["TokensInUse"])
                c["rep_queue_length"].append(r["QueueLength"]); c["rep_avg_input_tokens"].append(r["AvgInputTokens"])
                c["rep_avg_output_tokens"].append(r["AvgOutputTokens"]); c["rep_accelerator"].append(self.acc[r["AcceleratorName"]])
                c["rep_slot"].append(s)
                p = params.get((i["Namespace"], i["ModelID"], r["VariantName"])) or {}
                sB[s], sS[s] = p.get("EffectiveMaxBatchedTokens", 0), p.get("MaxNumSeqs", 0)
            off.append(len(c["rep_slot"]))
        return dict(c, model_replica_off=off, slot_max_batched_tokens=sB, slot_max_num_seqs=sS,
                    cfg_queue_threshold=[i["Config"]["QueueLengthThreshold"] for i in cycle],
                    cfg_kv_threshold=[i["Config"]["KvCacheThreshold"] for i in cycle])

    def history(self, count, values):
        """export (key order) -> {"model|acc|bucket": [values]}"""
        names = {v: k for k, v in self.acc.items()}
        out = {}
        for h, m in enumerate(self.hgs):
            for j in range(self.ao[h], self.ao[h + 1]):
                for b in range(3):
                    k = 3 * j + b
                    if count[k]:
                        out["%s|%s|%s" % (m, names[self.ai[j]], BUCKETS[b])] = [float(x) for x in values[k, :count[k]]]
        return out


def host_cycle(an, cycle, params):
    """phase 1 of SaturationAnalyzerV2.analyze_batch: the host chain, replica by replica; -1 (priority 4) -> k1"""
    k2 = []
    for i in cycle:
        for r in i["ReplicaMetrics"]:
            if r["TotalKvCapacityTokens"] <= 0:
                k2.append(-1)
                continue
            v = an._k2(i["ModelID"], r, i["Config"]["QueueLengthThreshold"], params.get((i["Namespace"], i["ModelID"], r["VariantName"])))
            x = float(r["TotalKvCapacityTokens"]) * i["Config"]["KvCacheThreshold"]
            k1 = int(x) if -9.2e18 < x < 9.2e18 else -(1 << 63)
            k2.append(v if v >= 0 else k1)
    return k2


# ---------------------------------------------------------------------------------------------------------------------
# seeded named sequences covering the cases of the chain
# ---------------------------------------------------------------------------------------------------------------------
AVG_OUT = (99.999, 100.0, 499.999, 500.0, float("nan"), 50.0, 250.0, 800.0, 0.0)
Q_THR = (5.0, 2.5, 0.0, -1.0, float("nan"), 3.7, 1e30)


def named_sequence(seed, n_cycles):
    rng = np.random.default_rng(seed)
    models = ["m%d" % k for k in range(3)]
    groups = []                                               # (model, namespace), a modelID in 1-5 namespaces
    for m in models:
        groups += [(m, "ns%d" % k) for k in range(int(rng.integers(1, 6)))]
    rng.shuffle(groups)
    cfg = {g: dict(CFG, QueueLengthThreshold=float(rng.choice(Q_THR)), KvCacheThreshold=float(rng.choice((0.8, 0.9, 0.5))))
           for g in groups}
    accs = ("H100", "A100", "")
    params = {}
    for (m, ns) in groups:
        for v in ("va", "vb", "vc"):
            if rng.random() < 0.5:
                params[(ns, m, v)] = {"EffectiveMaxBatchedTokens": int(rng.integers(512, 8192)), "MaxNumSeqs": int(rng.integers(16, 512))}
    cycles = []
    for _ in range(n_cycles):
        cyc = []
        for (m, ns) in groups:
            reps = []
            for k in range(int(rng.integers(0, 30 if rng.random() < 0.3 else 6))):
                v = str(rng.choice(("va", "vb", "vc")))
                cap = int(rng.choice((0, -5, 16000, 32000, 48000))) if rng.random() < 0.2 else int(rng.integers(1000, 50000))
                r = rm("p%d" % k, v, str(rng.choice(accs)), 1.0, int(rng.integers(0, 3) * rng.integers(0, 20000)), cap,
                       int(rng.integers(0, 12)), float(rng.choice((0.0, 100.0, 500.0, float(rng.uniform(0, 1000))))),
                       float(rng.choice(AVG_OUT)) if rng.random() < 0.5 else float(rng.uniform(0, 900)))
                r["ModelID"], r["Namespace"] = m, ns
                reps.append(r)
            states = [st(v, 1) for v in ("va", "vb") if rng.random() < 0.8]      # "vc" never has a state
            cyc.append({"ModelID": m, "Namespace": ns, "ReplicaMetrics": reps, "VariantStates": states,
                        "Config": cfg[(m, ns)], "SchedulerQueue": None})
        cycles.append(cyc)
    return cycles, params


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_oracle_and_host_chain_reproduce_reference_k2_cases(pkg, oracle):
    """analyzer_test.go:88-139 (history), :141-170 (output-length buckets), :172-224 (derived k2, k1 fallback)"""
    a1 = inp([rm("pod-1", "variant-a", "H100", 10.0, 8000, 16000, 6, 100, 50)], [st("variant-a", 1)])
    a2 = inp([rm("pod-1", "variant-a", "H100", 10.0, 6000, 16000, 2, 100, 50)], [st("variant-a", 1)])
    b2 = inp([rm("pod-1", "variant-a", "H100", 10.0, 6000, 16000, 2, 100, 600)], [st("variant-a", 1)])
    c1 = inp([rm("pod-1", "variant-a", "H100", 10.0, 5000, 16000, 2, 500, 100)], [st("variant-a", 1)])
    d1 = inp([rm("pod-1", "variant-a", "H100", 10.0, 5000, 16000, 0, 0, 0)], [st("variant-a", 1)])
    derived = {("test-ns", "test-model", "variant-a"): {"EffectiveMaxBatchedTokens": 2048, "MaxNumSeqs": 256}}
    cases = [([a1], {}, [8000], {"test-model|H100|short": [8000.0]}),           # observed, stored
             ([a1, a2], {}, [8000, 8000], {"test-model|H100|short": [8000.0]}),  # historical k2 = 8000, not k1 = 12800
             ([a1, b2], {}, [8000, 12800], {"test-model|H100|short": [8000.0]}), # no "long" history: k1
             ([c1], derived, [140800], {}),                                      # derived 256 * 550
             ([d1], {}, [12800], {})]                                            # k1 fallback
    for cycles, params, k2_want, hist_want in cases:
        cycles = [[c] for c in cycles]
        enc = Encoder(cycles)
        orc = K2Oracle(*enc.registry())
        an, chain = pkg.SaturationAnalyzerV2(OracleEngine(oracle)), pkg.SaturationAnalyzerV2(None)
        for (c,), want in zip(cycles, k2_want):
            assert orc.resolve(enc.columns([c], params))["rep_k2"].tolist() == [want]
            assert host_cycle(chain, [c], params) == [want]
            for (ns, m, v), p in params.items():
                an.store.update(ns, m, v, {"AcceleratorName": "H100", "GpuCount": 1, "VLLMParams": p, "LearnedFrom": "deployment"})
            res = an.analyze(c)
            assert res["VariantCapacities"][0]["PerReplicaCapacity"] == float(min(want, 12800))
        assert enc.history(*orc.export()) == hist_want
        assert an.history_state() == hist_want


@pytest.mark.parametrize("seed", range(4))
def test_oracle_matches_host_chain_over_cycles(pkg, seed):
    """30+ cycles: modelIDs in 1-5 namespaces with their own thresholds (fractional, NaN, negative), > 10 observations of
    a key in one cycle and across cycles, avgOutput at the bucket edges and NaN, replicas without capacity data,
    variants without state, accelerator ""; rep_k2 and the whole history after every cycle."""
    cycles, params = named_sequence(seed, 32)
    enc = Encoder(cycles)
    orc = K2Oracle(*enc.registry())
    an = pkg.SaturationAnalyzerV2(None)
    saw_many = False
    for cyc in cycles:
        o = orc.resolve(enc.columns(cyc, params))
        assert o is not None
        assert o["rep_k2"].tolist() == host_cycle(an, cyc, params)
        assert enc.history(*orc.export()) == an.history_state()
        saw_many |= any(len(v) == 10 for v in an.history.values())
    assert saw_many


def test_oracle_rejects_unregistered_accelerator_without_change():
    cycles, params = named_sequence(7, 3)
    enc = Encoder(cycles)
    orc = K2Oracle(*enc.registry())
    orc.resolve(enc.columns(cycles[0], params))
    before = orc.export()
    d = enc.columns(cycles[1], params)
    data = [k for k, t in enumerate(d["rep_total_kv_tokens"]) if t > 0]
    d["rep_accelerator"][data[0]] = 99
    assert orc.resolve(d) is None
    after = orc.export()
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1].view(np.int64), after[1].view(np.int64))


# ---------------------------------------------------------------------------------------------------------------------
# integer-level random registry + cycles (the GPU tests' scale)
# ---------------------------------------------------------------------------------------------------------------------
def int_registry(rng, G, wide=True):
    """history groups of 1-5 model groups, registry order shuffled; a few with 9-12 accelerators (more keys than a warp
    stages in shared memory)"""
    sizes = []
    while sum(sizes) < G:
        sizes.append(int(min(rng.integers(1, 6), G - sum(sizes))))
    H = len(sizes)
    perm = rng.permutation(G).astype(np.int32)
    mo = np.concatenate(([0], np.cumsum(sizes))).astype(np.int32)
    n_acc = rng.integers(1, 4, H)
    if wide:
        n_acc[rng.random(H) < 0.05] = 12
        n_acc[0] = 10
    ai = np.concatenate([rng.choice(16, int(k), replace=False) for k in n_acc]).astype(np.int32)
    ao = np.concatenate(([0], np.cumsum(n_acc))).astype(np.int32)
    return mo, perm, ao, ai, G * 4


def int_cycle(rng, reg, big_every=50):
    mo, mg, ao, ai, S = reg
    G = len(mg)
    hg_of = np.empty(G, np.int64)
    for h in range(len(mo) - 1):
        hg_of[mg[mo[h]:mo[h + 1]]] = h
    n = rng.integers(0, 9, G)
    n[::big_every] = rng.integers(33, 90, len(n[::big_every]))        # more than 32 data replicas per group
    off = np.concatenate(([0], np.cumsum(n))).astype(np.int32)
    P = int(off[-1])
    g_of = np.repeat(np.arange(G), n)
    h_of = hg_of[g_of]
    k = (rng.random(P) * (ao[h_of + 1] - ao[h_of])).astype(np.int64)
    acc = ai[ao[h_of] + k]
    tk = rng.integers(1000, 60000, P)
    tk[rng.random(P) < 0.15] = 0
    acc = np.where(tk > 0, acc, rng.integers(-3, 40, P)).astype(np.int32)   # not read without capacity data
    used = rng.integers(0, 20000, P) * (rng.random(P) < 0.9)
    ao_out = np.where(rng.random(P) < 0.3, np.array(AVG_OUT)[rng.integers(0, len(AVG_OUT), P)], rng.uniform(0, 900, P))
    q_thr = np.array(Q_THR)[rng.integers(0, len(Q_THR), G)]
    q_thr[rng.random(G) < 0.5] = 5.0
    return {"model_replica_off": off, "rep_total_kv_tokens": tk, "rep_tokens_in_use": used,
            "rep_queue_length": rng.integers(0, 9, P), "rep_avg_input_tokens": rng.uniform(0, 1000, P),
            "rep_avg_output_tokens": ao_out, "rep_accelerator": acc, "rep_slot": (g_of * 4 + rng.integers(0, 4, P)).astype(np.int32),
            "slot_max_batched_tokens": rng.integers(0, 8192, S) * (rng.random(S) < 0.5), "slot_max_num_seqs": rng.integers(1, 512, S),
            "cfg_queue_threshold": q_thr, "cfg_kv_threshold": rng.choice((0.8, 0.9, 0.5), G)}


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 1000, 100000])
def test_device_matches_oracle_bit_for_bit(pkg, engine, G):
    rng = np.random.default_rng(G)
    reg = int_registry(rng, G, wide=G > 1)
    orc = K2Oracle(*reg)
    with pkg.K2History(engine, *reg) as dev:
        assert dev.K == orc.K
        for cycle in range(20):
            d = int_cycle(rng, reg, big_every=1 if G == 1 else 50)
            P = len(d["rep_total_kv_tokens"])
            pos = np.where(rng.random(P) < 0.8, rng.permutation(P), -1).astype(np.int32)
            want = orc.resolve(d)
            got = dev.resolve(dict(d, rep_out_pos=pos, n_out=P))
            for k in ("rep_k2", "rep_effective", "slot_last_rep", "slot_effective"):
                assert np.array_equal(got[k], want[k]), (cycle, k)
            scat = np.full(P, -1, np.int64)
            scat[pos[pos >= 0]] = want["rep_k2"][pos >= 0]
            assert np.array_equal(got["out_rep_k2"], scat)
            e = dev.export()
            c, v = orc.export()
            assert np.array_equal(e["count"], c) and _bits_equal(e["values"], v), cycle
        assert (c == 10).any()                           # windows filled and rolled


@pytest.mark.gpu
def test_rejected_calls_leave_history_unchanged(pkg, engine):
    rng = np.random.default_rng(3)
    reg = int_registry(rng, 200)
    with pkg.K2History(engine, *reg) as dev:
        dev.resolve(int_cycle(rng, reg))
        before = dev.export()
        d = int_cycle(rng, reg)
        bad = dict(d, rep_accelerator=d["rep_accelerator"].copy())
        bad["rep_accelerator"][np.flatnonzero(d["rep_total_kv_tokens"] > 0)[-1]] = 999       # not registered
        off = d["model_replica_off"].copy()
        off[5] = off[-1] + 1                                                                  # not non-decreasing
        for case in (bad, dict(d, model_replica_off=off)):
            with pytest.raises(pkg.WvaError):
                dev.resolve(case)
            after = dev.export()
            assert np.array_equal(before["count"], after["count"]) and _bits_equal(before["values"], after["values"])
        with pytest.raises(pkg.WvaError):                                                     # duplicate key on import
            dev.import_({k: np.concatenate((v[:1], v[:1])) for k, v in before.items()})
        after = dev.export()
        assert np.array_equal(before["count"], after["count"]) and _bits_equal(before["values"], after["values"])


@pytest.mark.gpu
def test_export_import_resumes_like_an_uninterrupted_run(pkg, engine):
    rng = np.random.default_rng(11)
    reg = int_registry(rng, 2000)
    cycles = [int_cycle(rng, reg) for _ in range(12)]
    with pkg.K2History(engine, *reg) as a:
        outs_a = [a.resolve(c) for c in cycles]
        end_a = a.export()
    with pkg.K2History(engine, *reg) as b:
        outs_b = [b.resolve(c) for c in cycles[:5]]
        saved = b.export()
    with pkg.K2History(engine, *reg) as c:
        c.import_({k: v[saved["count"] > 0] for k, v in saved.items()})       # empty keys need not be listed
        outs_b += [c.resolve(x) for x in cycles[5:]]
        end_b = c.export()
    for x, y in zip(outs_a, outs_b):
        assert all(np.array_equal(x[k], y[k]) for k in x)
    assert np.array_equal(end_a["count"], end_b["count"]) and _bits_equal(end_a["values"], end_b["values"])


@pytest.mark.gpu
def test_analysis_runs_do_not_touch_history(pkg, engine):
    """wva_saturation_v2 as often as the caller likes after one resolve: the history moves only with wva_k2_resolve"""
    cycles, params = named_sequence(5, 4)
    an = pkg.SaturationAnalyzerV2(engine, device_history=True)
    try:
        for c in cycles[:3]:
            an.analyze_batch(c)
        before = an.k2.export()
        engine.saturation_v2(an.last_batch)
        engine.saturation_v2(an.last_batch)
        after = an.k2.export()
        assert np.array_equal(before["count"], after["count"]) and _bits_equal(before["values"], after["values"])
    finally:
        an.close()


def _fallback_sequence(seed, n):
    """named cycles where variants lose their ready replicas (zero-replica fallbacks read the store)"""
    cycles, params = named_sequence(seed, n)
    rng = np.random.default_rng(seed + 100)
    for k, cyc in enumerate(cycles):
        for i in cyc:
            i["VariantStates"] = [st("va", 1), st("vb", 2, pending=1)]
            if k % 3 == 2:                                   # "vb" has no ready replicas this cycle
                i["ReplicaMetrics"] = [r for r in i["ReplicaMetrics"] if r["VariantName"] != "vb"]
            if rng.random() < 0.2:
                i["ReplicaMetrics"] = []
    return cycles, params


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_analyzer_with_device_history_matches_host_history(pkg, engine, seed):
    cycles, params = _fallback_sequence(seed, 12)
    host, dev = pkg.SaturationAnalyzerV2(engine), pkg.SaturationAnalyzerV2(engine, device_history=True)
    try:
        for an in (host, dev):
            for (ns, m, v), p in params.items():
                an.store.update(ns, m, v, {"AcceleratorName": "H100", "GpuCount": 1, "VLLMParams": p, "LearnedFrom": "deployment",
                                           "EffectiveCapacity": 0, "TotalKvCapacityTokens": 0})
        for k, cyc in enumerate(cycles):
            if k == 6:                                         # a registry change in the middle: another list order
                cyc = cyc[::-1]
            rh, rd = host.analyze_batch(cyc), dev.analyze_batch(cyc)
            assert _same(rh, rd), k
            assert list(host.store.records.items()) == list(dev.store.records.items()), k
            assert host.history_state() == dev.history_state(), k
    finally:
        dev.close()


def _same(a, b):
    if isinstance(a, float) and isinstance(b, float):
        return (math.isnan(a) and math.isnan(b)) or a == b
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b
