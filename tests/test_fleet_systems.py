"""The sizer, both allocators, the grid and the sharded solve on fleet-shaped systems, against the oracle.

`synth.queue_system` (what the other parity tests size) gives every server its own model, at most 8 capacity types spread
evenly, no current allocations and three positive priorities.  A real fleet looks different, and so does the code that
serves it: a few models shared by many servers (per-model perf rows, some servers with an unknown model), up to 64
capacity types spread unevenly (the high half of the allocators' 64-bit type masks), more than 32 accelerators (the
allocators' candidate ranks past their 32-wide staging), current allocations (transition penalties decide the candidate
order and the greedy ties), keepAccelerator, many priority levels including negative ones and INT32_MAX.
`fleet_system` builds such systems and checks that each one really has that shape.
"""
import importlib
import os
import re
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "llm-d-workload-variant-autoscaler_b200"

INT_FIELDS = ("state", "num_replicas", "batch_size")
F32_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_arrv_rate")
SOL_INT = ("state", "acc", "num_replicas", "batch_size")
POLICIES = ("None", "PriorityExhaustive", "PriorityRoundRobin", "RoundRobin")
PRIORITY_LEVELS = np.array([-2**31, -7, -1, 0, 1, 2, 3, 5, 8, 10, 1000, 2**31 - 1], dtype=np.int64)
CUR_ACC_UNKNOWN = -2          # WVA_CUR_ACC_UNKNOWN: a current accelerator name that matches no accelerator


def _bit_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def fleet_system(S, M, A, T, seed, n_max=256, min_replicas=None, policy="None", delayed=False):
    """S servers sharing M models (Zipf-like, ~2 % unknown), A accelerators over T capacity types (uneven, one type
    without accelerators), perf data with holes and AccCount 0..8, ~70 % of the servers with a current allocation (a few
    on an unknown accelerator), ~15 % keepAccelerator, 12 priority levels, zero loads, TPS targets and unsatisfiable
    SLOs.  Every (model, accelerator) batch size and every server override stays <= n_max.  Unlimited capacity."""
    g = np.random.default_rng(seed)
    a = np.arange(A)
    # accelerator types: Zipf-like weights over a permutation of the types, one type left without accelerators
    w = 1.0 / (1.0 + np.arange(T)) ** 1.1
    w = w[g.permutation(T)]
    empty_type = int(g.integers(0, min(T, 32))) if T > 1 else -1
    if empty_type >= 0:
        w[empty_type] = 0.0
    acc_type = g.choice(T, A, p=w / w.sum())
    if T > 32:                                          # a quarter of the accelerators on the high half of the type masks
        acc_type[g.choice(A, A // 4, replace=False)] = g.integers(32, T, A // 4)
    d = {
        "n_acc": A, "n_types": T, "n_models": M, "n_servers": S,
        "acc_cost": (25.0 * 1.35 ** (a % 16) * (1 + a // 16)).astype(np.float32),
        "acc_multiplicity": g.choice(np.array([1, 2, 4, 8], np.int32), A),
        "acc_type": acc_type.astype(np.int32),
        "type_count": np.full(T, 2**31 - 1, dtype=np.int32),
    }
    # perf rows, one per model
    speed = (0.85 ** (a % 12))[None, :]
    d["perf_alpha"] = (g.uniform(4.0, 20.0, (M, A)) * speed).astype(np.float32)
    d["perf_beta"] = (g.uniform(0.01, 0.3, (M, A)) * speed).astype(np.float32)
    d["perf_gamma"] = (g.uniform(5e-4, 2e-2, (M, A)) * speed).astype(np.float32)
    mb = np.array([1, 4, 8, 16, 32, 64, 96, 128, 192, 256])
    mb = mb[mb <= n_max]
    d["perf_max_batch"] = g.choice(mb, (M, A)).astype(np.int32)
    d["perf_at_tokens"] = g.integers(8, 33, (M, A)).astype(np.int32)     # <= 32 <= AvgOutTokens: N <= MaxBatchSize
    d["perf_acc_count"] = g.integers(0, 9, (M, A)).astype(np.int32)
    d["perf_present"] = (g.random((M, A)) < 0.9).astype(np.uint8)
    # servers: models by a Zipf-like law, ~2 % unknown
    pm = 1.0 / (1.0 + np.arange(M)) ** 1.2
    model = g.permutation(M)[g.choice(M, S, p=pm / pm.sum())].astype(np.int32)
    model[g.random(S) < 0.02] = -1
    model[g.integers(0, S)] = -1
    in_tok = np.clip(np.floor(g.lognormal(np.log(512.0), 0.8, S)), 16, 8192).astype(np.int32)
    out_tok = np.clip(np.floor(g.lognormal(np.log(160.0), 0.7, S)), 32, 2048).astype(np.int32)
    arrival = 60.0 * np.exp(g.uniform(np.log(0.05), np.log(60.0), S))
    arrival[(g.random(S) < 0.05) | (np.arange(S) == S // 2)] = 0.0
    cls = g.integers(0, 3, S)
    slo = np.array([(500.0, 24.0, 0.0), (2000.0, 80.0, 0.0), (0.0, 200.0, 0.0)])[cls] * g.uniform(0.8, 1.25, S)[:, None]
    tps = (g.random(S) < 0.1) | (np.arange(S) == 1)
    slo[tps, 2] = g.uniform(50.0, 3000.0, int(tps.sum()))
    slo[g.random(S) < 0.02, 1] = 0.01                   # unsatisfiable ITL
    max_batch = np.zeros(S, np.int32)
    mbs = (g.random(S) < 0.05) | (np.arange(S) == 2)
    max_batch[mbs] = g.integers(1, n_max + 1, int(mbs.sum()))
    # current allocations: ~70 % on a known accelerator, a few on an unknown one, ~15 % keepAccelerator
    cur = np.full(S, -1, np.int32)
    has = g.random(S) < 0.7
    cur[has] = g.integers(0, A, int(has.sum()))
    unk = (g.random(S) < 0.02) | (np.arange(S) == 3)
    cur[unk] = CUR_ACC_UNKNOWN
    cur_rep = np.where(cur != -1, g.integers(1, 7, S), 0).astype(np.int32)
    mult = d["acc_multiplicity"][np.maximum(cur, 0)]
    cur_cost = np.where(cur >= 0, d["acc_cost"][np.maximum(cur, 0)] * cur_rep * mult * g.uniform(0.8, 1.2, S),
                        np.where(cur == CUR_ACC_UNKNOWN, 100.0 * cur_rep, 0.0)).astype(np.float32)
    keep = ((g.random(S) < 0.15) | (np.arange(S) == 4)).astype(np.uint8)
    prio = g.choice(PRIORITY_LEVELS, S)
    prio[5:7] = PRIORITY_LEVELS[[1, -1]]                # a negative level and INT32_MAX in every system
    minr = g.integers(0, 4, S) if min_replicas is None else np.full(S, min_replicas)
    if min_replicas is None:
        minr[S // 2] = 0                                # zero load, no replicas: the empty allocation
    d.update({
        "srv_model": model,
        "srv_priority": prio.astype(np.int32),
        "srv_min_replicas": minr.astype(np.int32),
        "srv_max_batch": max_batch,
        "srv_keep_acc": keep,
        "srv_target_present": np.ones(S, np.uint8),
        "srv_slo_ttft": slo[:, 0].astype(np.float32),
        "srv_slo_itl": slo[:, 1].astype(np.float32),
        "srv_slo_tps": slo[:, 2].astype(np.float32),
        "srv_arrival": arrival.astype(np.float32),
        "srv_in_tokens": in_tok, "srv_out_tokens": out_tok,
        "srv_cur_acc": cur, "srv_cur_replicas": cur_rep, "srv_cur_cost": cur_cost,
        "unlimited": True, "delayed_best_effort": delayed, "saturation_policy": policy,
    })
    _assert_fleet_shape(d)
    return d


def _assert_fleet_shape(d):
    """the system really is fleet-shaped (and not a queue_system in disguise)"""
    S, A, T, M = d["n_servers"], d["n_acc"], d["n_types"], d["n_models"]
    known = d["srv_model"] >= 0
    assert len(np.unique(d["srv_model"][known])) < S / 4 and (~known).any()
    counts = np.bincount(d["acc_type"], minlength=T)
    assert (counts == 0).any() and counts.max() >= min(3, A)
    if T > 32:
        assert (d["acc_type"] >= 32).any()
    assert set(np.unique(d["perf_acc_count"])) >= {0, 8} and not d["perf_present"].all()
    assert (d["srv_cur_acc"] >= 0).any() and (d["srv_cur_acc"] == CUR_ACC_UNKNOWN).any() and d["srv_keep_acc"].any()
    assert (d["srv_priority"] < 0).any() and (d["srv_priority"] == 2**31 - 1).any()
    assert (d["srv_arrival"] == 0).any() and (d["srv_slo_tps"] > 0).any() and (d["srv_max_batch"] > 0).any()
    if A > 32:   # a server that can have more than 32 candidates: known model, > 32 accelerators with perf data, not pinned
        npres = d["perf_present"].astype(np.int64).sum(axis=1)[np.maximum(d["srv_model"], 0)]
        assert (known & (npres > 32) & ((d["srv_keep_acc"] == 0) | (d["srv_cur_acc"] == -1))).any()


def _assert_fleet_candidates(d, cand):
    """candidates that carry a transition penalty (value != cost on a server with a current allocation) and, with more
    than 32 accelerators, a server with more than 32 of them"""
    st = np.asarray(cand["state"])
    has_cur = (d["srv_cur_acc"] != -1)[:, None]
    pen = (st == 1) & has_cur & (np.asarray(cand["value"]) != np.asarray(cand["cost"]))
    assert pen.sum() >= 10, pen.sum()
    assert (st[d["srv_model"] < 0] == 0).all()
    if d["n_acc"] > 32:
        assert ((st != 0).sum(axis=1) > 32).any()


# ---- generator (CPU) ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,M,A,T", [(120, 10, 12, 9), (200, 16, 40, 33), (200, 16, 96, 64)])
def test_fleet_generator_shape(oracle, S, M, A, T):
    d = fleet_system(S, M, A, T, seed=S + A + T)
    cand = oracle.calculate(d)
    _assert_fleet_candidates(d, cand)
    assert (np.asarray(cand["state"]) == 1).any() and (np.asarray(cand["state"]) == 2).any()


# ---- sharding with unknown and shared models (CPU) -----------------------------------------------------------------------
def test_shard_system_keeps_unknown_models_unknown(pkg):
    """a shard holds each of its servers' models once; a server of unknown model stays unknown (no perf row)"""
    d = fleet_system(90, 8, 10, 9, seed=11)
    for world in (2, 3):
        for rank in range(world):
            sd, idx = pkg.synth.shard_system(d, rank, world)
            whole = d["srv_model"][idx]
            assert np.array_equal(sd["srv_model"] < 0, whole < 0)
            known = whole >= 0
            assert sd["n_models"] == len(np.unique(whole[known]))
            for k in ("perf_alpha", "perf_max_batch", "perf_acc_count", "perf_present"):
                mine = np.asarray(sd[k]).reshape(sd["n_models"], d["n_acc"])[sd["srv_model"][known]]
                assert np.array_equal(mine, np.asarray(d[k]).reshape(d["n_models"], d["n_acc"])[whole[known]]), k


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


# (policy, delayedBestEffort); policy None is also run with unlimited capacity (SolveUnlimited)
SHARD_CASES = (("unlimited", False), ("None", False), ("PriorityExhaustive", False), ("PriorityRoundRobin", True),
               ("RoundRobin", False))


def _limited_fleet(pkg_synth, orc, policy, delayed):
    d = fleet_system(61, 6, 10, 9, seed=29, policy="None" if policy == "unlimited" else policy, delayed=delayed)
    if policy == "unlimited":
        return d
    un = orc.solve(d, orc.calculate(d, nthreads=1))
    return pkg_synth.limit_capacity(d, un["type_count"], 0.5)


def _shard_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    pkg_synth = importlib.import_module(PKG + ".synth")
    sharding = importlib.import_module(PKG + ".sharding")
    from tests import oracle_lib
    from tests.test_distributed_cpu import _OracleEngine
    orc = oracle_lib.load()
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        out = []
        for policy, delayed in SHARD_CASES:
            d = _limited_fleet(pkg_synth, orc, policy, delayed)
            sol = sharding.solve_sharded(_OracleEngine(orc), d, rank, world)
            out.append({k: np.asarray(v) for k, v in sol.items()})
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_fleet_solve_equals_whole_gloo(pkg, oracle, world):
    """sharding.solve_sharded over gloo with the oracle standing in for the device, on a fleet system (shared models,
    unknown-model servers, current allocations, limited capacity): every rank ends with the whole system's solution."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for i, (policy, delayed) in enumerate(SHARD_CASES):
        d = _limited_fleet(pkg.synth, oracle, policy, delayed)
        ref = oracle.solve(d, oracle.calculate(d))
        assert (np.asarray(ref["state"]) == 1).any() and (np.asarray(ref["state"]) == 0).any()
        assert (np.asarray(ref["state"])[d["srv_model"] < 0] == 0).all()
        for r in range(world):
            for k, v in ref.items():
                assert _bit_equal(np.asarray(got[r][i][k]), np.asarray(v)), (policy, r, k)


# ---- device: sizer ---------------------------------------------------------------------------------------------------
def _cmp_candidates_bits(g, o, what=""):
    for k in INT_FIELDS:
        assert np.array_equal(g[k], o[k]), (k, what, np.argwhere(np.asarray(g[k]) != np.asarray(o[k]))[:5])
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), (k, what)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["warp", "lane", "pool"])
def test_fleet_calculate_matches_oracle(engine, oracle, size):
    """System.Calculate on fleet systems, every field bit for bit, at one size per default sizer: a small system (warp
    per pair), a mid-size one (lane per pair) and one above 640 pairs per SM (pool sizer)."""
    if size == "warp":
        d, want = fleet_system(100, 10, 12, 9, seed=101), (1,)
    elif size == "lane":
        d, want = fleet_system(400, 30, 40, 33, seed=102), (2, 3)
    else:
        A = 40
        d, want = fleet_system(640 * _sm_count() // A + 100, 60, A, 40, seed=103), (4,)
    engine.load_system(d)
    engine.calculate()
    g = engine.candidates()
    assert engine.timing()["sizer_kernel"] in want, (engine.timing()["sizer_kernel"], want)
    o = oracle.calculate(d)
    _cmp_candidates_bits(g, o, size)
    _assert_fleet_candidates(d, o)


@pytest.mark.gpu
def test_fleet_calculate_every_lane_mode_and_table_mode(engine, oracle):
    """the same system through every lane sizer mode (WVA_OPT_FORCE_LANE_SIZER 1..6) and both head-table placements"""
    d = fleet_system(300, 24, 16, 12, seed=104)
    o = oracle.calculate(d)
    for mode, table in [(1, 0), (2, 0), (3, 0), (4, 0), (5, 0), (6, 0), (2, 1), (2, 2)]:
        engine.set_option(1, mode); engine.set_option(4, table)
        try:
            engine.load_system(d); engine.calculate()
            g = engine.candidates()
        finally:
            engine.set_option(1, 0); engine.set_option(4, 0)
        _cmp_candidates_bits(g, o, (mode, table))


# ---- device: unlimited solve and by-type totals ---------------------------------------------------------------------------
def _by_type(d, sol):
    """AllocateByType restated on the host: replicas x AccCount of the server's MODEL (<= 0 -> 1) x multiplicity"""
    tc = np.zeros(d["n_types"], np.int64)
    inst = np.maximum(np.asarray(d["perf_acc_count"]).reshape(d["n_models"], d["n_acc"]), 1)
    for i in np.flatnonzero((sol["state"] == 1) & (d["srv_model"] >= 0)):
        a = sol["acc"][i]
        tc[d["acc_type"][a]] += int(sol["num_replicas"][i]) * int(inst[d["srv_model"][i], a]) * int(d["acc_multiplicity"][a])
    return tc


@pytest.mark.gpu
@pytest.mark.parametrize("T,A", [(9, 12), (33, 40), (64, 64), (64, 96)])
def test_fleet_unlimited_solve_matches_oracle(engine, oracle, T, A):
    d = fleet_system(300, 20, A, T, seed=200 + T + A)
    engine.load_system(d); engine.calculate()
    g = engine.candidates()
    o = oracle.calculate(d)
    _cmp_candidates_bits(g, o)
    engine.solve()
    sol = engine.solution()
    osol = oracle.solve(d, o)
    for k in ("state", "acc", "num_replicas"):
        assert np.array_equal(sol[k], osol[k]), k
    assert np.array_equal(sol["type_count"], osol["type_count"])
    assert np.array_equal(sol["type_count"], _by_type(d, osol))
    np.testing.assert_allclose(sol["type_cost"], osol["type_cost"], rtol=1e-12)
    if T > 32:
        assert sol["type_count"][32:].sum() > 0


# ---- device: SolveGreedy, both formulations ---------------------------------------------------------------------------------
def _limited(pkg, d, demand, frac, zero_types=()):
    assert np.asarray(demand).max() < 2**31
    lim = pkg.synth.limit_capacity(d, demand, frac)
    lim["type_count"] = lim["type_count"].copy()
    lim["type_count"][list(zero_types)] = 0
    return lim


def _greedy_vs_oracle(engine, oracle, lim, cand, policy, delayed, mode, ocache):
    """re-solve the loaded system under another capacity / OptimizerSpec / formulation; the oracle's greedy takes the
    device's candidates (the sizer has its own parity tests)"""
    lim = dict(lim, saturation_policy=policy, delayed_best_effort=delayed)
    engine.set_option(5, mode)
    try:
        engine.set_capacity(lim["type_count"]); engine.set_optimizer(False, delayed, policy)
        engine.solve()
        g = engine.solution()
    finally:
        engine.set_option(5, 0)
    key = (lim["type_count"].tobytes(), policy, delayed)
    if key not in ocache:
        ocache[key] = oracle.solve(lim, cand)
    o = ocache[key]
    for k in SOL_INT:
        assert np.array_equal(g[k], o[k]), (k, policy, delayed, mode, np.argwhere(g[k] != o[k])[:5])
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), (k, policy, delayed, mode)
    assert np.array_equal(g["type_count"], o["type_count"]) and (g["type_count"] <= lim["type_count"]).all()
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("T,A", [(9, 12), (32, 32), (33, 40), (64, 64), (64, 96)])
def test_fleet_greedy_matches_oracle(pkg, engine, oracle, T, A):
    """every policy x delayedBestEffort at 30 % and 60 % of the unlimited demand, two populated types without capacity,
    in the default formulation, the literal queue (WVA_OPT_GREEDY_MODE 1) and the event sweep (2)"""
    d = fleet_system(500, 30, A, T, seed=300 + T + A)
    engine.load_system(d); engine.calculate()
    cand = engine.candidates()
    engine.set_optimizer(True); engine.solve()
    un = engine.solution()
    present = np.flatnonzero(un["type_count"] > 0)
    zero = present[np.argsort(un["type_count"][present])[[0, len(present) // 2]]]
    ocache, binds = {}, False
    for frac in (0.3, 0.6):
        lim = _limited(pkg, d, un["type_count"], frac, zero)
        for mode in (0, 1, 2):
            for policy in POLICIES:
                for delayed in (False, True):
                    g = _greedy_vs_oracle(engine, oracle, lim, cand, policy, delayed, mode, ocache)
                    binds |= (g["state"] == 0).sum() > (un["state"] == 0).sum()
                    assert (g["type_count"][zero] == 0).all()
    assert binds


@pytest.mark.gpu
def test_fleet_greedy_nothing_fits_on_the_high_types(pkg, engine, oracle, capfd, monkeypatch):
    """Every type below 32 has no capacity and every server wants >= 3 replicas: the sweep reaches the point where no
    remaining candidate fits while single replicas still fit on types >= 32 only, so bestEffort's survivors are decided by
    the high half of the type masks (g_live_types) and the nothing-fits test by the high half of the block minima.  Every
    policy, both formulations, against the oracle; the debug line proves that the case with survivors was exercised."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    d = fleet_system(600, 40, 64, 64, seed=401, min_replicas=3)
    engine.load_system(d); engine.calculate()
    cand = engine.candidates()
    engine.set_optimizer(True); engine.solve()
    un = engine.solution()
    ocache, survivors = {}, []
    for frac in (0.2, 0.35, 0.5, 0.65):
        lim = _limited(pkg, d, un["type_count"], frac, range(32))
        for mode in (2, 1):
            for policy, delayed in (("None", False), ("PriorityExhaustive", False), ("PriorityExhaustive", True),
                                    ("PriorityRoundRobin", False), ("PriorityRoundRobin", True), ("RoundRobin", False),
                                    ("RoundRobin", True)):
                capfd.readouterr()
                g = _greedy_vs_oracle(engine, oracle, lim, cand, policy, delayed, mode, ocache)
                err = capfd.readouterr().err
                assert (g["state"] == 1).any() and (d["acc_type"][g["acc"][g["state"] == 1]] >= 32).all()
                if mode == 2:
                    survivors += [int(x) for x in re.findall(r"after nothing fits: (-?\d+)", err)]
    assert any(x > 0 for x in survivors), sorted(set(survivors))


@pytest.mark.gpu
def test_fleet_greedy_20k_servers_64_types(pkg, engine, oracle):
    """20 000 servers x 40 accelerators over 64 types (pool sizer; the sweep's block-minimum rows span many blocks):
    the sizer and the unlimited solve against the oracle, then every policy at 50 % of the demand in both formulations."""
    d = fleet_system(20_000, 200, 40, 64, seed=501, n_max=64)
    engine.load_system(d); engine.calculate()
    cand = engine.candidates()
    _cmp_candidates_bits(cand, oracle.calculate(d))
    engine.set_optimizer(True); engine.solve()
    un = engine.solution()
    osol = oracle.solve(d, cand)
    for k in ("state", "acc", "num_replicas"):
        assert np.array_equal(un[k], osol[k]), k
    assert np.array_equal(un["type_count"], osol["type_count"])
    present = np.flatnonzero(un["type_count"] > 0)
    lim = _limited(pkg, d, un["type_count"], 0.5, present[:1])
    ocache = {}
    for policy, delayed in (("None", False), ("PriorityExhaustive", False), ("PriorityRoundRobin", True),
                            ("RoundRobin", False)):
        for mode in (0, 1):
            g = _greedy_vs_oracle(engine, oracle, lim, cand, policy, delayed, mode, ocache)
            assert (g["state"] == 0).sum() > (un["state"] == 0).sum()


# ---- device: replica grid --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("defer", [1, 2])
def test_fleet_grid_matches_oracle(engine, oracle, defer):
    """the replica grid reads per-model perf rows: a materialised grid and a frontier-only run on fleet systems, with and
    without the deferred near-saturation pass"""
    d = fleet_system(60, 8, 12, 9, seed=601, n_max=128)
    R = 40
    o = oracle.analyze_grid(d, R)
    big = fleet_system(300, 20, 40, 33, seed=602)
    ofr = oracle.analyze_grid(big, 64, full=False)["frontier"]
    engine.set_option(6, defer)
    try:
        engine.load_system(d)
        g = engine.analyze_grid(R)
        engine.grid_run(R, full=False)
        fr = engine.grid_fetch_frontier()
        engine.load_system(big)
        engine.grid_run(64, full=False)
        bfr = engine.grid_fetch_frontier()
    finally:
        engine.set_option(6, 0)
    assert np.array_equal(g["ok"], o["ok"]) and np.array_equal(g["frontier"], o["frontier"])
    assert np.array_equal(fr, o["frontier"]) and np.array_equal(bfr, ofr)
    for k in ("ttft", "itl", "rho", "tput"):
        assert _bit_equal(g[k], o[k]), k
    assert (o["ok"][d["srv_model"] < 0] == 0).all() and o["ok"].any() and (ofr > 0).any()


# ---- device: boundaries ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_64_types_load_and_65_do_not(pkg, engine, oracle):
    d = fleet_system(80, 8, 70, 64, seed=701)
    sol = engine.optimize(d)
    osol = oracle.solve(d, oracle.calculate(d))
    for k in ("state", "acc", "num_replicas"):
        assert np.array_equal(sol[k], osol[k]), k
    assert np.array_equal(sol["type_count"], osol["type_count"])
    with pytest.raises(pkg.WvaError, match="size exceeds kernel limits.*64 capacity types"):
        engine.load_system(fleet_system(80, 8, 70, 65, seed=702))
    sol2 = engine.optimize(d)                      # the refused load left the context usable
    assert np.array_equal(sol2["acc"], sol["acc"])


# ---- device: sharded limited solve ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy,delayed", [("None", False), ("PriorityRoundRobin", True), ("RoundRobin", False)])
def test_sharded_fleet_limited_solve_equals_whole(pkg, engine, oracle, policy, delayed):
    """as test_gpu_parity.py::test_sharded_limited_solve_equals_whole, on a fleet system: the shards of a 3-rank partition
    (shared models, unknown-model servers) are sized one after the other and merged; the candidates and the greedy sweep
    on the merged set equal the whole system's, bit for bit"""
    sh = pkg.sharding
    d = fleet_system(301, 20, 16, 12, seed=801, policy=policy, delayed=delayed)
    engine.load_system(d); engine.calculate(); engine.solve()
    lim = pkg.synth.limit_capacity(d, engine.solution()["type_count"], 0.55)
    engine.load_system(lim); engine.calculate()
    whole_c = engine.candidates(); engine.solve(); whole = engine.solution()
    world, S, A = 3, 301, 16
    rows = (S + world - 1) // world
    full = {k: np.zeros((S, A), dt) for k, dt in sh._CAND_FIELDS}
    for r in range(world):
        shard, idx = pkg.synth.shard_system(lim, r, world)
        assert shard["n_models"] < len(idx) and (shard["srv_model"] < 0).any()
        engine.load_system(shard); engine.calculate()
        part = sh.unpack_candidates(sh.pack_candidates(engine.candidates(), rows, A), rows, A)
        for k in full:
            full[k][idx] = part[k][: len(idx)]
    for k, _ in sh._CAND_FIELDS:
        if k != "n_solves":
            assert np.array_equal(full[k].view(np.uint8), np.asarray(whole_c[k]).view(np.uint8)), k
    engine.load_system(lim); engine.set_candidates(full); engine.solve()
    merged = engine.solution()
    o = oracle.solve(lim, whole_c)
    for k in SOL_INT:
        assert np.array_equal(merged[k], whole[k]) and np.array_equal(merged[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(merged[k], whole[k]) and _bit_equal(merged[k], o[k]), k
    assert np.array_equal(merged["type_count"], whole["type_count"]) and (whole["state"] == 0).any()
