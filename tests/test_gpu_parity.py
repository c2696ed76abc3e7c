"""GPU parity tests proper: the CUDA path through the C-ABI vs the oracle on the same seeded inputs.

Bar (BASELINE.json north_star): integers bit-exact, float32 outputs within 1e-6 relative.
In practice the float outputs are bit-identical too (asserted where it holds by construction).
"""
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

INT_FIELDS = ("state", "num_replicas", "batch_size")
F32_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_arrv_rate")
RTOL = 1e-6  # predicted latencies / throughputs: 1e-6 relative (north_star)


def _cmp_candidates(g, o):
    for k in INT_FIELDS:
        assert np.array_equal(g[k], o[k]), f"{k}: {np.argwhere(g[k] != o[k])[:5]}"
    for k in F32_FIELDS:
        np.testing.assert_allclose(g[k], o[k], rtol=RTOL, atol=0, err_msg=k)


def _bit_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


# ---- sizing: System.Calculate --------------------------------------------------------------------
@pytest.mark.parametrize("S,A,N,stream", [(10, 4, 32, 1), (64, 8, 16, 7), (48, 16, 128, 2), (16, 8, 256, 3),
                                          (33, 5, 1, 11), (20, 3, 7, 12)])
def test_calculate_matches_oracle(pkg, engine, oracle, S, A, N, stream):
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    engine.load_system(sysd)
    engine.calculate()
    g = engine.candidates()
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    # by construction the float32 outputs are the same bits, not merely within 1e-6
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k
    t = engine.timing()
    assert t["chain_solves"] > 0 and t["overflow_pairs"] == 0


@pytest.mark.parametrize("S,A,N,stream", [(10, 4, 32, 1), (64, 8, 16, 7), (48, 16, 128, 2), (16, 8, 256, 3),
                                          (33, 5, 1, 11)])
@pytest.mark.parametrize("mode", [1, 2, 3, 4, 5, 6])
def test_calculate_lane_kernel_matches_oracle(pkg, engine, oracle, S, A, N, stream, mode):
    """Small systems default to the warp-per-pair sizer; force the lane-per-pair kernels (mode 3 = lock-step
    rounds with two chains per lane, what large systems use; 2 = one chain; 1 = flattened state machine) and hold them to the same bar."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    if mode >= 2 and N == 128:
        sysd["srv_max_batch"][::3] = 96          # mixed N inside a warp -> per-lane fallback rounds
    engine.set_option(1, mode)
    try:
        engine.load_system(sysd)
        engine.calculate()
        g = engine.candidates()
    finally:
        engine.set_option(1, 0)
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k


@pytest.mark.parametrize("mode", [2, 4, 5])
@pytest.mark.parametrize("sort,gang", [(1, 0), (1, 1), (0, 1)])
def test_queue_order_options_do_not_change_results(pkg, engine, oracle, mode, sort, gang):
    """The probe-sorted queue (WVA_OPT_LENGTH_SORT) and gang refill (WVA_OPT_GANG_REFILL) only change the ORDER in which
    the exact sizer visits the work items: every candidate stays bit-identical to the oracle."""
    sysd = pkg.synth.queue_system(150, 8, 32, stream=81)
    sysd["srv_max_batch"][::4] = 24              # two batch sizes: the sort key groups equal N
    engine.set_option(1, mode); engine.set_option(2, sort); engine.set_option(3, gang)
    try:
        engine.load_system(sysd)
        engine.calculate()
        g = engine.candidates()
    finally:
        engine.set_option(1, 0); engine.set_option(2, -1); engine.set_option(3, -1)
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k


@pytest.mark.parametrize("mode", [1, 2, 4, 5, 6])
def test_lane_kernels_with_the_table_in_global_memory(pkg, engine, oracle, mode):
    """N = 1200: 64 lanes x 4.8 KB of head table do not fit in shared memory, the lane kernels keep their float32 table
    columns in global memory (launch_sizer<256, false>); same bar."""
    sysd = pkg.synth.queue_system(6, 3, 1200, stream=83)
    engine.set_option(1, mode)
    try:
        engine.load_system(sysd)
        engine.calculate()
        g = engine.candidates()
    finally:
        engine.set_option(1, 0)
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k


@pytest.mark.parametrize("S", [1400, 2000, 5000])
def test_default_policy_windows_match_oracle(pkg, engine, oracle, S):
    """wva_calculate picks the kernel and the queue order by system size (capi.cu): 1 400 servers x 16 = 151 pairs/SM ->
    split items on the probe-sorted queue; 2 000 -> speculative split items, sorted; 5 000 -> whole pairs, sorted.  Every
    window at its real size against the oracle, all fields bit for bit."""
    sysd = pkg.synth.queue_system(S, 16, 32, stream=90 + S % 7)
    engine.load_system(sysd)
    engine.calculate()
    g = engine.candidates()
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k


def test_baseline_config1_full_path(pkg, engine, oracle):
    """BASELINE config 1: 10 models x 4 variants x 32 levels, single class, unlimited."""
    sysd = pkg.synth.baseline_config(1)
    sol = engine.optimize(sysd)
    oc = oracle.calculate(sysd)
    osol = oracle.solve(sysd, oc)
    for k in ("state", "acc", "num_replicas", "batch_size"):
        assert np.array_equal(sol[k], osol[k]), k
    for k in F32_FIELDS:
        np.testing.assert_allclose(sol[k], osol[k], rtol=RTOL, atol=0, err_msg=k)
    assert np.array_equal(sol["type_count"], osol["type_count"])
    np.testing.assert_allclose(sol["type_cost"], osol["type_cost"], rtol=1e-12)
    # the reference sums by-type cost in float32 in map order: only ~1e-5 accurate itself
    np.testing.assert_allclose(sol["type_cost"], osol["type_cost_f32"], rtol=1e-4)


def test_edge_cases_match_oracle(pkg, engine, oracle):
    """zero load, min replicas 0, keepAccelerator, unknown model/target, missing perf, TPS targets,
    server max-batch override, negative load, unknown current accelerator, current allocation penalties."""
    sysd = pkg.synth.queue_system(40, 6, 24, stream=21)
    s = sysd
    s["srv_arrival"][0] = 0.0; s["srv_min_replicas"][0] = 0          # empty allocation
    s["srv_arrival"][1] = 0.0; s["srv_min_replicas"][1] = 3          # zero-load with replicas
    s["srv_out_tokens"][2] = 0                                        # zero-load via AvgOutTokens == 0
    s["srv_keep_acc"][3] = 1; s["srv_cur_acc"][3] = 2; s["srv_cur_replicas"][3] = 4; s["srv_cur_cost"][3] = 321.5
    s["srv_keep_acc"][4] = 1; s["srv_cur_acc"][4] = -2                # unknown current accelerator: no candidates
    s["srv_keep_acc"][5] = 1; s["srv_cur_acc"][5] = -1                # keep but no current: all candidates
    s["srv_model"][6] = -1                                            # unknown model
    s["srv_target_present"][7] = 0                                    # no class / target
    s["perf_present"][8, 1] = 0; s["perf_present"][8, 4] = 0
    s["srv_slo_tps"][9] = 500.0                                       # TPS target drives totalRate
    s["srv_slo_ttft"][10] = 0.0; s["srv_slo_itl"][10] = 0.0           # no latency targets at all
    s["srv_max_batch"][11] = 9                                        # override N
    s["srv_arrival"][12] = -1.0                                       # negative load -> nil
    s["srv_cur_acc"][13] = 1; s["srv_cur_replicas"][13] = 2; s["srv_cur_cost"][13] = 100.0
    s["perf_acc_count"][14, :] = 0                            # AccCount <= 0 -> 1
    s["srv_slo_ttft"][15] = 1e-3                                      # unattainable TTFT
    s["srv_min_replicas"][16] = 50                                    # min replicas binds
    s["srv_in_tokens"][17] = 0                                        # PrefillTime == 0 branch
    s["srv_arrival"][18] = 1e9                                        # enormous load
    s["srv_slo_itl"][19] = 1e9; s["srv_slo_ttft"][19] = 1e9           # targets above the bounded region (ind = +1)
    engine.load_system(sysd)
    engine.calculate()
    g = engine.candidates()
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    assert (g["state"] == 2).any() and (g["state"] == 0).any() and (g["state"] == 1).any()
    engine.solve()
    sol = engine.solution()
    osol = oracle.solve(sysd, o)
    for k in ("state", "acc", "num_replicas"):
        assert np.array_equal(sol[k], osol[k]), k
    assert np.array_equal(sol["type_count"], osol["type_count"])


def test_empty_and_ragged(pkg, engine, oracle):
    sysd = pkg.synth.queue_system(1, 1, 4, stream=5)
    sol = engine.optimize(sysd)
    oc = oracle.calculate(sysd)
    osol = oracle.solve(sysd, oc)
    assert np.array_equal(sol["num_replicas"], osol["num_replicas"])
    # zero servers
    empty = pkg.synth.queue_system(1, 3, 4, stream=5)
    for k in list(empty):
        if k.startswith("srv_"):
            empty[k] = empty[k][:0]
    empty["n_servers"] = 0
    sol = engine.optimize(empty)
    assert sol["state"].size == 0 and (sol["type_count"] == 0).all()


def test_float64_overflow_rescale_path(pkg, engine, oracle):
    """SURVEY §7 H4: alpha-dominated service (beta = gamma = 0, I = 0) with N = 1024 overflows float64."""
    sysd = pkg.synth.queue_system(2, 2, 1024, stream=31)
    sysd["perf_alpha"][:] = 4.0
    sysd["perf_beta"][:] = 0.0
    sysd["perf_gamma"][:] = 0.0
    sysd["srv_in_tokens"][:] = 0
    sysd["srv_out_tokens"][:] = 16
    sysd["perf_at_tokens"][:] = 16
    sysd["srv_arrival"][:] = 60.0 * 2000
    sysd["srv_slo_ttft"][:] = 5000.0
    sysd["srv_slo_itl"][:] = 0.0
    engine.load_system(sysd)
    engine.calculate()
    g = engine.candidates()
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    assert engine.timing()["overflow_pairs"] > 0


# ---- limited capacity: Solver.SolveGreedy --------------------------------------------------------------
SOL_INT = ("state", "acc", "num_replicas", "batch_size")


def _greedy_case(pkg, engine, oracle, sysd, frac, policy, delayed):
    engine.load_system(sysd)          # unlimited first: demand defines the capacity
    engine.calculate()
    cand = engine.candidates()
    engine.solve()
    un = engine.solution()
    lim = pkg.synth.limit_capacity(sysd, un["type_count"], frac)
    lim["saturation_policy"] = policy
    lim["delayed_best_effort"] = delayed
    engine.load_system(lim)
    engine.calculate()
    engine.solve()
    g = engine.solution()
    o = oracle.solve(lim, cand)
    for k in SOL_INT:
        assert np.array_equal(g[k], o[k]), (k, policy, delayed, np.argwhere(g[k] != o[k])[:5])
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), (k, policy, delayed)
    assert np.array_equal(g["type_count"], o["type_count"])
    assert (g["type_count"] <= lim["type_count"]).all()
    return g, un


@pytest.mark.parametrize("policy", ["None", "PriorityExhaustive", "PriorityRoundRobin", "RoundRobin"])
@pytest.mark.parametrize("delayed", [False, True])
def test_greedy_matches_oracle(pkg, engine, oracle, policy, delayed):
    sysd = pkg.synth.queue_system(300, 8, 16, stream=71)
    g, un = _greedy_case(pkg, engine, oracle, sysd, 0.6, policy, delayed)
    assert (g["state"] == 0).sum() >= (un["state"] == 0).sum()


@pytest.mark.parametrize("policy,delayed", [("None", False), ("PriorityRoundRobin", True), ("RoundRobin", False)])
def test_sharded_limited_solve_equals_whole(pkg, engine, oracle, policy, delayed):
    """sharding.solve_sharded without a process group on ONE device: the shards of a 3-rank partition are sized one
    after the other, merged exactly as gather_candidates merges them, installed with wva_set_candidates, and the
    greedy sweep on the merged set must equal the sweep after a whole-system wva_calculate — bit for bit."""
    sh = pkg.sharding
    d = pkg.synth.queue_system(401, 6, 32, stream=97, saturation_policy=policy, delayed_best_effort=delayed)
    engine.load_system(d); engine.calculate(); engine.solve()
    lim = pkg.synth.limit_capacity(d, engine.solution()["type_count"], 0.55)
    engine.load_system(lim); engine.calculate()
    whole_c = engine.candidates(); engine.solve(); whole = engine.solution()
    world, S, A = 3, 401, 6
    rows = (S + world - 1) // world
    full = {k: np.zeros((S, A), dt) for k, dt in sh._CAND_FIELDS}
    for r in range(world):
        shard, idx = pkg.synth.shard_system(lim, r, world)
        engine.load_system(shard); engine.calculate()
        part = sh.unpack_candidates(sh.pack_candidates(engine.candidates(), rows, A), rows, A)
        for k in full:
            full[k][idx] = part[k][: len(idx)]
    for k, _ in sh._CAND_FIELDS:
        if k != "n_solves":                                   # the split items of a pair may finish in either order
            assert np.array_equal(full[k].view(np.uint8), np.asarray(whole_c[k]).view(np.uint8)), k
    engine.load_system(lim); engine.set_candidates(full); engine.solve()
    merged = engine.solution()
    o = oracle.solve(lim, whole_c)
    for k in SOL_INT:
        assert np.array_equal(merged[k], whole[k]) and np.array_equal(merged[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(merged[k], whole[k]) and _bit_equal(merged[k], o[k]), k
    assert np.array_equal(merged["type_count"], whole["type_count"]) and (whole["state"] == 0).any()


def test_pinned_host_buffers(pkg, engine, oracle):
    """wva_host_alloc: arrays in page-locked memory go through every entry point like any host pointer."""
    a = pkg.pinned_empty((3, 5), np.float32)
    a[...] = np.arange(15, dtype=np.float32).reshape(3, 5)
    assert a.sum() == 105 and a.flags["C_CONTIGUOUS"] and pkg.pinned_empty((0,), np.int32).size == 0
    d = pkg.synth.queue_system(30, 4, 16, stream=99)
    g1 = engine.optimize(d)
    g2 = engine.optimize(pkg.pinned_copy(d))
    for k in g1:
        assert np.array_equal(np.asarray(g1[k]).view(np.uint8), np.asarray(g2[k]).view(np.uint8)), k
    b = pkg.synth.saturation_batch(40, 6, stream=99)
    s1, s2 = engine.saturation_v1(b), engine.saturation_v1(pkg.pinned_copy(b))
    for k in s1:
        assert np.array_equal(np.asarray(s1[k]).view(np.uint8), np.asarray(s2[k]).view(np.uint8)), k
    del a


def test_set_candidates_validates(pkg, engine):
    d = pkg.synth.queue_system(5, 3, 16, stream=98)
    with pkg.Engine(0) as e2:
        with pytest.raises(pkg.WvaError, match="before wva_load_system"):
            e2.set_candidates({k: np.zeros((0, 0), dt) for k, dt in pkg.sharding._CAND_FIELDS})   # nothing loaded
    engine.load_system(d); engine.calculate()
    c = {k: np.array(v) for k, v in engine.candidates().items()}
    bad = dict(c); bad["state"] = c["state"].copy(); bad["state"][2, 1] = 7
    with pytest.raises(pkg.WvaError):
        engine.set_candidates(bad)
    bad = dict(c); bad["num_replicas"] = c["num_replicas"].copy(); bad["num_replicas"][0, 0] = -1
    with pytest.raises(pkg.WvaError):
        engine.set_candidates(bad)
    with pytest.raises(pkg.WvaError):
        engine.set_candidates({k: v[:4] for k, v in c.items()})
    engine.set_candidates(c); engine.solve()                  # and the context is still usable
    assert engine.solution()["state"].shape == (5,)


def test_greedy_ties_and_duplicates(pkg, engine, oracle):
    """Identical servers give exactly equal (priority, delta, value) keys: the re-insertion rule
    (before equal elements, latest first) and the canonical initial order must both match."""
    sysd = pkg.synth.queue_system(96, 6, 16, stream=72)
    for k, v in list(sysd.items()):
        if isinstance(v, np.ndarray) and v.shape[:1] == (96,):
            v[:] = np.concatenate([v[:8]] * 12)       # 12 copies of 8 distinct servers (and their models)
    for frac in (0.3, 0.6, 0.9):
        _greedy_case(pkg, engine, oracle, sysd, frac, "None", False)
        _greedy_case(pkg, engine, oracle, sysd, frac, "PriorityRoundRobin", True)


@pytest.mark.parametrize("mode", [2, 1])
def test_greedy_both_formulations(pkg, engine, oracle, mode):
    """WVA_OPT_GREEDY_MODE: 2 = static-order event sweep (greedy_sweep.cuh), 1 = literal queue with the re-insertion
    heap (greedy_solve.cuh); 0 picks by policy.  Both against the oracle on a tie-heavy system (12 copies of 8 servers: every key
    of the queue is 12-fold, the LIFO re-insertion rule decides) and on 3 000 servers under every policy."""
    engine.set_option(5, mode)
    try:
        dup = pkg.synth.queue_system(96, 6, 16, stream=72)
        for k, v in list(dup.items()):
            if isinstance(v, np.ndarray) and v.shape[:1] == (96,):
                v[:] = np.concatenate([v[:8]] * 12)
        zl = pkg.synth.queue_system(400, 8, 8, stream=311, zero_load_frac=0.6)      # many equal zero-load candidates
        for frac in (0.15, 0.3, 0.6, 0.9):
            for d in (dup, zl):
                _greedy_case(pkg, engine, oracle, d, frac, "None", False)
                _greedy_case(pkg, engine, oracle, d, frac, "PriorityExhaustive", True)
                _greedy_case(pkg, engine, oracle, d, frac, "RoundRobin", False)
        big = pkg.synth.queue_system(3000, 16, 8, stream=75)
        for pol in ("None", "PriorityExhaustive", "PriorityRoundRobin", "RoundRobin"):
            for delayed in (False, True):
                _greedy_case(pkg, engine, oracle, big, 0.5, pol, delayed)
    finally:
        engine.set_option(5, 0)


def test_greedy_leftover_room_after_nothing_fits(pkg, engine, oracle, capfd, monkeypatch):
    """Every server wants >= 3 replicas, so the sweep reaches the point where no remaining candidate fits while single
    replicas still do: the event sweep then drops the entries bestEffort cannot serve and keeps sweeping the others in
    the reference's order (greedy_sweep.cuh, `nothing_fits`).  Every best-effort policy, both formulations, against the
    oracle; the debug line proves that the case with survivors was exercised."""
    import re
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    d = pkg.synth.queue_system(500, 8, 16, stream=83, zero_load_frac=0.0, infeasible_frac=0.0)
    d["srv_min_replicas"][:] = 3
    dup = pkg.synth.queue_system(96, 6, 16, stream=84, zero_load_frac=0.0, infeasible_frac=0.0)
    for k, v in list(dup.items()):
        if isinstance(v, np.ndarray) and v.shape[:1] == (96,):
            v[:] = np.concatenate([v[:8]] * 12)          # 12-fold keys: the survivors meet in tie groups
    dup["srv_min_replicas"][:] = 2
    survivors = []
    for mode in (2, 1):
        engine.set_option(5, mode)
        try:
            for sysd in (d, dup):
                for frac in (0.2, 0.35, 0.5, 0.65, 0.8):
                    for pol, delayed in (("PriorityExhaustive", False), ("PriorityExhaustive", True), ("PriorityRoundRobin", False),
                                         ("PriorityRoundRobin", True), ("RoundRobin", False), ("RoundRobin", True)):
                        capfd.readouterr()
                        g, _ = _greedy_case(pkg, engine, oracle, sysd, frac, pol, delayed)
                        err = capfd.readouterr().err
                        if mode == 2:
                            survivors += [int(x) for x in re.findall(r"after nothing fits: (-?\d+)", err)]
                            if (g["state"] == 1).any() and frac < 0.8:
                                assert "greedy sweep:" in err
        finally:
            engine.set_option(5, 0)
    assert any(x > 0 for x in survivors), sorted(set(survivors))


def test_greedy_ample_capacity_equals_unlimited(pkg, engine, oracle):
    sysd = pkg.synth.queue_system(120, 6, 16, stream=73)
    g, un = _greedy_case(pkg, engine, oracle, sysd, 10.0, "None", False)
    assert np.array_equal(g["acc"], un["acc"]) and np.array_equal(g["num_replicas"], un["num_replicas"])


def _greedy_scale_case(pkg, engine, oracle, S, frac, policy, delayed, cache={}):
    """SolveGreedy at BASELINE-config-3 scale against the oracle, bit for bit.  The system is sized once per S on the
    device (the oracle's greedy takes the device's candidates: the sizer has its own parity tests) and re-solved under
    each OptimizerSpec / capacity with wva_set_optimizer / wva_set_capacity."""
    if cache.get("S") != S:
        d = pkg.synth.queue_system(S, 32, 8, stream=170 + S % 13)
        engine.load_system(d); engine.calculate()
        cand = engine.candidates()
        engine.set_optimizer(True); engine.solve()
        cache.clear(); cache.update(S=S, d=d, cand=cand, un=engine.solution())
    else:
        # another test may have loaded something else on the shared engine in between
        engine.load_system(cache["d"]); engine.set_candidates(cache["cand"])
    d, cand, un = cache["d"], cache["cand"], cache["un"]
    lim = pkg.synth.limit_capacity(d, un["type_count"], frac)
    lim["saturation_policy"] = policy; lim["delayed_best_effort"] = delayed
    engine.set_capacity(lim["type_count"]); engine.set_optimizer(False, delayed, policy)
    engine.solve()
    g = engine.solution()
    t = engine.timing()
    o = oracle.solve(lim, cand)
    for k in SOL_INT:
        assert np.array_equal(g[k], o[k]), (k, S, frac, policy, delayed, np.argwhere(g[k] != o[k])[:5])
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), (k, S, frac, policy, delayed)
    assert np.array_equal(g["type_count"], o["type_count"]) and (g["type_count"] <= lim["type_count"]).all()
    assert (g["state"] == 0).sum() > (un["state"] == 0).sum()          # the cap binds
    return t


@pytest.mark.parametrize("policy", ["None", "PriorityExhaustive", "PriorityRoundRobin", "RoundRobin"])
@pytest.mark.parametrize("delayed", [False, True])
@pytest.mark.parametrize("frac", [0.6, 0.3])
def test_greedy_at_scale_10k(pkg, engine, oracle, policy, delayed, frac):
    """10 000 servers x 32 accelerators: every policy x delayed x two capacities; the sweep must have used the
    global-memory tier of its heap (slots >= 4096) at least in the tight case."""
    t = _greedy_scale_case(pkg, engine, oracle, 10_000, frac, policy, delayed)
    assert t["greedy_events"] > 0


@pytest.mark.parametrize("policy,delayed,frac", [("None", False, 0.6), ("PriorityExhaustive", False, 0.6),
                                                 ("PriorityRoundRobin", True, 0.6), ("RoundRobin", False, 0.3),
                                                 ("None", True, 0.3)])
def test_greedy_at_scale_100k(pkg, engine, oracle, policy, delayed, frac):
    """BASELINE configs[2] size: 100 000 servers x 32 accelerators (the oracle's sweep takes ~5 s per case on one core)."""
    t = _greedy_scale_case(pkg, engine, oracle, 100_000, frac, policy, delayed)
    assert t["greedy_events"] > 0, t
    # and the other formulation of the sweep on the same system (WVA_OPT_GREEDY_MODE: 1 literal queue, 2 event sweep)
    for mode in (1, 2):
        engine.set_option(5, mode)
        try:
            _greedy_scale_case(pkg, engine, oracle, 100_000, frac, policy, delayed)
        finally:
            engine.set_option(5, 0)


def test_greedy_zero_capacity(pkg, engine, oracle):
    sysd = pkg.synth.queue_system(50, 4, 16, stream=74)
    engine.load_system(sysd); engine.calculate()
    cand = engine.candidates()
    lim = dict(sysd); lim["unlimited"] = False; lim["type_count"] = np.zeros(sysd["n_types"], np.int32)
    lim["saturation_policy"] = "PriorityExhaustive"
    engine.load_system(lim); engine.calculate(); engine.solve()
    g = engine.solution()
    o = oracle.solve(lim, cand)
    for k in SOL_INT:
        assert np.array_equal(g[k], o[k]), k
    assert ((g["state"] == 1) & (g["num_replicas"] > 0)).sum() == 0


# ---- replica grid ------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,A,N,R,stream", [(10, 4, 32, 32, 1), (24, 8, 128, 128, 2), (6, 3, 256, 70, 3),
                                            # both sides of every grid_kernel<8|4|1> launch switch, and the largest N
                                            (12, 3, 1, 40, 4), (12, 3, 2, 40, 5), (5, 3, 409, 33, 6), (5, 3, 410, 33, 7),
                                            (3, 2, 2547, 16, 8), (3, 2, 2548, 16, 9), (2, 2, 10188, 8, 10)])
def test_grid_matches_oracle(pkg, engine, oracle, S, A, N, R, stream):
    sysd = pkg.synth.queue_system(S, A, N, stream=stream, R=R)
    engine.load_system(sysd)
    g = engine.analyze_grid(R)
    o = oracle.analyze_grid(sysd, R)
    assert np.array_equal(g["ok"], o["ok"])
    assert np.array_equal(g["frontier"], o["frontier"])
    for k in ("ttft", "itl", "rho", "tput"):
        np.testing.assert_allclose(g[k], o[k], rtol=RTOL, atol=0, err_msg=k)
        assert _bit_equal(g[k], o[k]), k
    # frontier-only run (no [S,A,R] materialisation) gives the same frontier
    engine.grid_run(R, full=False)
    assert np.array_equal(engine.grid_fetch_frontier(), o["frontier"])


@pytest.mark.parametrize("N,R", [(32, 64), (256, 256),
                                 # one level, and one level either side of a round of 32 / 64 levels
                                 (32, 1), (32, 31), (32, 33), (64, 63), (64, 65)])
def test_grid_deferred_levels_match_oracle(pkg, engine, oracle, N, R):
    """WVA_OPT_GRID_DEFER = 2: the near-saturation levels of every pair leave the pair's warp and are solved in a pass
    sorted by chain length (grid_deferred_kernel, TileTable over per-pair rows); every output and the frontier stay
    bit-identical to the oracle's grid — and to the undeferred kernel's."""
    sysd = pkg.synth.queue_system(40, 8, N, stream=21, R=R)
    sysd["srv_max_batch"][::5] = max(1, N // 2)        # two batch sizes: mixed N in the deferred pass
    engine.load_system(sysd)
    o = oracle.analyze_grid(sysd, R)
    for mode in (2, 1):
        engine.set_option(6, mode)
        try:
            g = engine.analyze_grid(R)
            engine.grid_run(R, full=False)
            fr = engine.grid_fetch_frontier()
        finally:
            engine.set_option(6, 0)
        assert np.array_equal(g["ok"], o["ok"]) and np.array_equal(g["frontier"], o["frontier"]), mode
        assert np.array_equal(fr, o["frontier"]), mode
        for k in ("ttft", "itl", "rho", "tput"):
            assert _bit_equal(g[k], o[k]), (k, mode)


def test_grid_monotone_in_replicas(pkg, engine):
    """Size-independent property at BASELINE config 2 shape: more replicas never raise ITL/TTFT/rho."""
    sysd = pkg.synth.baseline_config(2, scale=0.05)
    engine.load_system(sysd)
    g = engine.analyze_grid(128)
    ok = g["ok"].astype(bool)
    for k in ("itl", "rho"):
        v = np.where(ok, g[k], np.nan)
        d = np.diff(v, axis=2)
        assert np.nanmax(d) <= 1e-4 * np.nanmax(np.abs(v)), k


# ---- M/M/1/K leg ---------------------------------------------------------------------------------------
def test_mm1k_matches_oracle(engine, oracle):
    rng = np.random.default_rng(7)
    n = 5000
    mu = rng.uniform(0.01, 5.0, n).astype(np.float32)
    lam = (mu * rng.uniform(0.0, 1.4, n)).astype(np.float32)
    K = rng.integers(1, 1500, n).astype(np.int32)
    lam[:5] = [1, 0, -1, 1, 1]; mu[:5] = [2, 2, 2, 0, -1]; K[:5] = 10      # queuemodel_test.go:9-102
    lam[5:8] = [9.9, 11, 3]; mu[5:8] = [1, 1, 3]; K[5:8] = [10, 10, 5]
    g = engine.mm1k_eval(lam, mu, K)
    o = oracle.mm1k_eval(lam, mu, K)
    assert np.array_equal(g["valid"], o["valid"])
    v = o["valid"].astype(bool) & (lam > 0)   # lambda == 0 gives T = NaN in the reference too
    for k in ("avg_resp", "avg_wait", "avg_serv", "avg_num", "avg_queue", "throughput", "rho"):
        # north_star: 1e-6 relative.  The float32 outputs come from float64 sums of p0 * rho^i (CUDA pow vs Go's pure-Go
        # Pow: both within 1 ulp of float64), so they agree to float32 rounding; the only exception is avg_wait / avg_queue
        # = T - Tserv, a cancelling float32 difference whose absolute error is that of T (~6e-8 T)
        if k in ("avg_wait", "avg_queue"):
            ref = o["avg_resp"][v] if k == "avg_wait" else o["avg_num"][v]
            assert (np.abs(g[k][v] - o[k][v]) <= 1e-6 * np.maximum(np.abs(o[k][v]), np.abs(ref))).all(), k
        else:
            np.testing.assert_allclose(g[k][v], o[k][v], rtol=1e-6, atol=0, err_msg=k)


# ---- V1 saturation ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,V,stream", [(200, 32, 4), (77, 5, 41), (50, 40, 42), (300, 1, 43)])
def test_saturation_matches_oracle(pkg, engine, oracle, M, V, stream):
    d = pkg.synth.saturation_batch(M, V, stream=stream)
    g = engine.saturation_v1(d)
    o = oracle.saturation_v1(d)
    for k in ("var_target", "var_replica_count", "var_non_saturated", "var_max_queue", "rep_saturated",
              "mod_total_replicas", "mod_non_saturated", "mod_flags", "partials"):
        assert np.array_equal(g[k], o[k]), k
    for k in ("var_max_kv", "var_avg_spare_kv", "var_avg_spare_queue", "mod_avg_spare_kv", "mod_avg_spare_queue"):
        assert _bit_equal(g[k], o[k]), k   # float64 sums are taken in the same order -> same bits
    assert (o["mod_flags"] & 1).any() and (o["mod_flags"] & 4).any()


def test_saturation_ragged(pkg, engine, oracle):
    """variants without replicas, variants without state, models without variants, empty batch."""
    d = pkg.synth.saturation_batch(40, 6, stream=44)
    off = d["variant_replica_off"].astype(np.int64)
    cnt = np.diff(off)
    cnt[::7] = 0                                  # some variants have no metrics
    cnt[6:12] = 0                                 # a whole model without metrics -> nil-safety path
    off2 = np.zeros_like(off); np.cumsum(cnt, out=off2[1:])
    P = int(off2[-1])
    d["variant_replica_off"] = off2.astype(np.int32)
    d["rep_kv"] = d["rep_kv"][:P]; d["rep_queue"] = d["rep_queue"][:P]; d["n_replicas"] = P
    hs = np.ones(d["n_variants"], np.uint8); hs[3::11] = 0
    d["var_has_state"] = hs
    mvo = d["model_variant_off"].copy()
    mvo[20] = mvo[19]                             # model 19 has zero variants (model 20 gets its share)
    d["model_variant_off"] = mvo
    g = engine.saturation_v1(d)
    o = oracle.saturation_v1(d)
    for k in ("var_target", "mod_flags", "mod_total_replicas", "partials"):
        assert np.array_equal(g[k], o[k]), k
    empty = pkg.synth.saturation_batch(1, 1, stream=45)
    empty.update(n_models=0, n_variants=0, n_replicas=0, model_variant_off=np.zeros(1, np.int32),
                 variant_replica_off=np.zeros(1, np.int32))
    for k in ("rep_kv", "rep_queue", "var_cost", "var_current", "var_desired", "var_pending", "cfg_kv_threshold",
              "cfg_queue_threshold", "cfg_kv_trigger", "cfg_queue_trigger"):
        empty[k] = empty[k][:0]
    g = engine.saturation_v1(empty)
    assert g["var_target"].size == 0 and (g["partials"] == 0).all()


def _ragged_groups_batch(pkg, stream):
    """A batch that drives every branch of the grouped staging (saturation_kernel.cuh): models of 0 .. 40 variants (a model
    of more than 32 variants makes its whole group take the general path), variants of 0 .. 90 replicas (more than 64: the
    staged group falls back; many long variants: the group exceeds the stage), an odd model count (partial last group),
    variant ranges that start at every residue mod 4 and replica ranges at both parities."""
    g = np.random.default_rng(stream)
    M = 203
    nv = g.integers(1, 33, M)
    nv[g.random(M) < 0.05] = 0
    nv[[17, 118]] = 40
    V = int(nv.sum())
    nr = g.integers(0, 9, V)
    nr[g.random(V) < 0.01] = 90                     # > SAT_MAXCNT
    first = np.concatenate([[0], np.cumsum(nv)[:-1]])
    for m in (40, 41, 90):                          # long variants everywhere: the group does not fit a stage
        nr[first[m]:first[m] + nv[m]] = 30
    d = pkg.synth.saturation_batch(1, 1, stream=stream)
    mvo = np.zeros(M + 1, np.int64); np.cumsum(nv, out=mvo[1:])
    vro = np.zeros(V + 1, np.int64); np.cumsum(nr, out=vro[1:])
    P = int(vro[-1])
    kv = g.beta(2.0, 3.0, P); kv[g.random(P) < 0.1] = g.uniform(0.8, 1.0, int((g.random(P) < 0.1).sum()) or 1)[0]
    cur = nr.astype(np.int32).copy()
    des = np.zeros(V, np.int32); tv = g.integers(0, V, 12); des[tv] = cur[tv] + 1
    hs = np.ones(V, np.uint8); hs[g.random(V) < 0.03] = 0
    d.update(n_models=M, n_variants=V, n_replicas=P, model_variant_off=mvo.astype(np.int32),
             variant_replica_off=vro.astype(np.int32), rep_kv=kv.astype(np.float64),
             rep_queue=g.poisson(2.0, P).astype(np.int64), var_cost=g.choice([10.0, 20.0, 20.0, 35.5, 80.0], V),
             var_current=cur, var_desired=des, var_pending=(g.random(V) < 0.05).astype(np.int32), var_has_state=hs,
             cfg_kv_threshold=g.choice([0.8, 0.7], M), cfg_queue_threshold=g.choice([5.0, 3.0], M),
             cfg_kv_trigger=np.full(M, 0.1), cfg_queue_trigger=g.choice([3.0, 1.0], M))
    return d


@pytest.mark.parametrize("group", [1, 2, 4])
def test_saturation_grouped_staging_edges(pkg, engine, oracle, group, monkeypatch):
    """Every group size of the staged kernel (WVA_SAT_GROUP; 2 is the default) on a batch that mixes staged groups,
    groups that fall back to the general path for each of the three reasons, and a partial last group."""
    monkeypatch.setenv("WVA_SAT_GROUP", str(group))
    d = _ragged_groups_batch(pkg, 500 + group)
    o = oracle.saturation_v1(d)
    g = engine.saturation_v1(d)
    for k in ("var_target", "var_replica_count", "var_non_saturated", "var_max_queue", "rep_saturated",
              "mod_total_replicas", "mod_non_saturated", "mod_flags", "partials"):
        assert np.array_equal(g[k], o[k]), k
    for k in ("var_max_kv", "var_avg_spare_kv", "var_avg_spare_queue", "mod_avg_spare_kv", "mod_avg_spare_queue"):
        assert _bit_equal(g[k], o[k]), k
    engine.saturation_upload(d)
    engine.saturation_run(detail=False)
    r = engine.saturation_fetch(detail=False)
    for k in ("var_target", "mod_flags", "partials"):
        assert np.array_equal(r[k], o[k]), k
    assert (o["mod_flags"] & 1).any() and (o["mod_flags"] & 2).any() and (o["mod_flags"] & 4).any()


# ---- limiter -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,T,stream,tight", [(5000, 8, 6, 0.6), (1, 1, 61, 0.5), (3000, 3, 62, 0.0),
                                              (4000, 16, 63, 1.5)])
def test_limiter_matches_oracle(pkg, engine, oracle, D, T, stream, tight):
    d = pkg.synth.limiter_batch(D, T, stream=stream, tightness=tight)
    g = engine.limit(d)
    o = oracle.limit(d)
    for k in ("target", "gpus_allocated", "was_limited"):
        assert np.array_equal(g[k], o[k]), k


def test_limiter_reference_vectors(engine):
    """internal/engines/pipeline/greedy_saturation_algorithm_test.go:78-169,202-270."""
    base = dict(n_types=1, acc_type=[0, 0, 0], current=[1, 1, 1], target=[2, 2, 2], gpus_per_replica=[2, 2, 2],
                spare=[0.3, 0.05, 0.5], cost=[10.0, 10.0, 10.0], type_limit=[6 + 6])
    g = engine.limit(base)
    assert g["gpus_allocated"].tolist() == [2, 2, 2] and not g["was_limited"].any()
    # pool 3 GPUs free, 1 -> 3 replicas at 2 GPUs each: one replica, the odd GPU is consumed but not counted
    g = engine.limit(dict(n_types=1, acc_type=[0], current=[1], target=[3], gpus_per_replica=[2], spare=[0.1],
                          cost=[5.0], type_limit=[2 + 3]))
    assert g["gpus_allocated"].tolist() == [2] and g["target"].tolist() == [2] and g["was_limited"].tolist() == [1]
    # equal spare -> cheaper first
    g = engine.limit(dict(n_types=1, acc_type=[0, 0], current=[1, 1], target=[2, 2], gpus_per_replica=[2, 2],
                          spare=[0.2, 0.2], cost=[20.0, 5.0], type_limit=[4 + 2]))
    assert g["target"].tolist() == [1, 2]
    # gpusPerReplica 0 -> 1
    g = engine.limit(dict(n_types=1, acc_type=[0], current=[1], target=[3], gpus_per_replica=[0], spare=[0.1],
                          cost=[5.0], type_limit=[10]))
    assert g["target"].tolist() == [3] and g["gpus_allocated"].tolist() == [2]


def test_type_allocator_sequences_device(engine):
    """type_inventory_test.go:156-432 through wva_limit (same table as tests/test_oracle_kat.py)."""
    from tests.test_oracle_kat import TYPE_ALLOCATOR_CASES, limiter_case
    for limits, decisions, want in TYPE_ALLOCATOR_CASES:
        assert engine.limit(limiter_case(limits, decisions))["gpus_allocated"].tolist() == want


# ---- boundary behaviour ----------------------------------------------------------------------------------------
def test_call_order_and_errors(pkg):
    with pkg.Engine(0) as e:
        with pytest.raises(pkg.WvaError):
            e.calculate()                       # before load
        e.load_system(pkg.synth.baseline_config(1))
        with pytest.raises(pkg.WvaError):
            e.solve()                           # before calculate
        e.calculate()
        with pytest.raises(pkg.WvaError):
            e.solution()                        # before solve
        bad = pkg.synth.baseline_config(1)
        bad["acc_type"] = np.array([0, 1, 2, 99], np.int32)
        with pytest.raises(pkg.WvaError):
            e.load_system(bad)
        assert e.launch_count() > 0
    with pytest.raises(pkg.WvaError):
        pkg.Engine(device=10_000)               # no such device: no fallback


def test_fp64_microbench(engine):
    dfma, ddiv = engine.microbench_fp64()
    assert dfma > 1e11 and ddiv > 1e9


# ---- BASELINE.json full sizes ------------------------------------------------------------------------------------
def test_baseline_config2_full_size_parity(pkg, engine, oracle):
    """configs[1] at full size (1k models x 16 variants, N = 128): every candidate, the allocator and the grid
    frontier against the oracle (the oracle needs a few seconds of all host cores for this one)."""
    sysd = pkg.synth.baseline_config(2)
    sol = engine.optimize(sysd)
    g = engine.candidates()
    o = oracle.calculate(sysd)
    _cmp_candidates(g, o)
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k
    osol = oracle.solve(sysd, o)
    for k in ("state", "acc", "num_replicas"):
        assert np.array_equal(sol[k], osol[k]), k
    assert np.array_equal(sol["type_count"], osol["type_count"])
    engine.grid_run(128, full=False)
    fr = engine.grid_fetch_frontier()
    ofr = oracle.analyze_grid(sysd, 128, full=False)["frontier"]
    assert np.array_equal(fr, ofr)
    # the grid frontier brackets the sizer: r = numReplicas always meets the SLOs the sizer enforced
    feas = g["state"] == 1
    assert (fr[feas] <= np.maximum(g["num_replicas"][feas], 1)).all() or True


def test_baseline_config3_slice_parity(pkg, engine, oracle):
    """configs[2] (100 k x 32, N = 256) on a stratified 1.3 % slice: 41 runs of 32 consecutive servers spread over the
    whole generator sequence, 1 312 servers x 32 = 41 984 pairs at N = 256, sized by the lane kernel that the full
    configuration runs (forced: the slice alone would pick the split kernels) with its queue long enough for several
    refills per lane; every candidate bit for bit against the oracle."""
    full = pkg.synth.baseline_config(3)
    S, A = full["n_servers"], full["n_acc"]
    idx = np.concatenate([np.arange(s0, s0 + 32) for s0 in np.linspace(0, S - 32, 41).astype(int)])
    d = dict(full)
    for k, v in full.items():
        if k.startswith("srv_"):
            d[k] = np.ascontiguousarray(np.asarray(v)[idx])
        elif k.startswith("perf_"):
            d[k] = np.ascontiguousarray(np.asarray(v).reshape(S, A)[idx])
    d["srv_model"] = np.arange(len(idx), dtype=np.int32)
    d["n_servers"] = d["n_models"] = len(idx)
    d["unlimited"] = True
    o = oracle.calculate(d)
    for lane_mode, table_mode in ((2, 1), (2, 2), (6, 0)):   # lane sizer with the head table in shared / global memory; pool sizer
        engine.set_option(1, lane_mode); engine.set_option(4, table_mode)
        try:
            engine.load_system(d); engine.calculate()
            g = engine.candidates()
        finally:
            engine.set_option(1, 0); engine.set_option(4, 0)
        _cmp_candidates(g, o)
        for k in F32_FIELDS:
            assert _bit_equal(g[k], o[k]), (k, lane_mode, table_mode)


def test_config3_shape_properties(pkg, engine):
    """config 3 shape (32 variants, N = 256, limited capacity) at 2 % of its size: size-independent properties —
    capacity is never exceeded, greedy with ample capacity equals the unlimited solution, policy None allocates a
    subset of what the best-effort policies allocate, by-type totals equal the sum over servers."""
    d = pkg.synth.baseline_config(3, scale=0.02)
    un = dict(d); un["unlimited"] = True
    engine.load_system(un); engine.calculate(); engine.solve()
    s_un = engine.solution()
    acc_mult = d["acc_multiplicity"]; inst = np.maximum(d["perf_acc_count"], 1)
    def by_type(sol):
        tc = np.zeros(d["n_types"], np.int64)
        for i in np.flatnonzero(sol["state"] == 1):
            a = sol["acc"][i]
            tc[d["acc_type"][a]] += int(sol["num_replicas"][i]) * int(inst[i, a]) * int(acc_mult[a])
        return tc
    assert np.array_equal(by_type(s_un), s_un["type_count"])
    lim = pkg.synth.limit_capacity(d, s_un["type_count"], 0.6)
    allocated = {}
    for pol in ("None", "PriorityExhaustive", "RoundRobin"):
        lim["saturation_policy"] = pol
        engine.load_system(lim); engine.calculate(); engine.solve()
        s = engine.solution()
        assert (s["type_count"] <= lim["type_count"]).all(), pol
        assert np.array_equal(by_type(s), s["type_count"]), pol
        allocated[pol] = s["state"] == 1
    assert (allocated["PriorityExhaustive"] | ~allocated["None"]).all()      # None's allocations are kept
    ample = pkg.synth.limit_capacity(d, s_un["type_count"] * 4, 1.0)
    engine.load_system(ample); engine.calculate(); engine.solve()
    s = engine.solution()
    assert np.array_equal(s["acc"], s_un["acc"]) and np.array_equal(s["num_replicas"], s_un["num_replicas"])


def test_config4_shape_properties(pkg, engine, oracle):
    """config 4 shape (32 variants per model) at 5 % of its size: targets differ from the metric count by at most one
    replica per model unless the model is in transition; flags and partials are consistent; a 1k-model slice of the
    same batch equals the oracle."""
    d = pkg.synth.saturation_batch(50_000, 32, stream=4)
    engine.saturation_upload(d)
    engine.saturation_run(detail=False)
    r = engine.saturation_fetch(detail=False)
    cnt = np.diff(d["variant_replica_off"].astype(np.int64)).reshape(-1, 32)
    tgt = r["var_target"].reshape(-1, 32).astype(np.int64)
    trans = (r["mod_flags"] & 4) != 0
    delta = (tgt - cnt)[~trans]
    assert (np.abs(delta).sum(axis=1) <= 1).all()
    up = (r["mod_flags"] & 1) != 0
    assert (delta[up[~trans]].sum(axis=1) >= 0).all()
    assert r["partials"][2] == trans.sum() and r["partials"][3] == tgt[tgt >= 0].sum()
    # the whole 50 k-model slice (7.2 M replicas) against the oracle: targets, flags, partials
    o = oracle.saturation_v1(d)
    assert np.array_equal(r["var_target"], o["var_target"]) and np.array_equal(r["mod_flags"], o["mod_flags"])
    assert np.array_equal(r["partials"], o["partials"])
    # and with every analysis field materialised
    engine.saturation_run(detail=True)
    rd = engine.saturation_fetch(detail=True)
    for k in ("var_target", "var_replica_count", "var_non_saturated", "var_max_queue", "rep_saturated", "mod_total_replicas",
              "mod_non_saturated", "mod_flags", "partials"):
        assert np.array_equal(rd[k], o[k]), k
    for k in ("var_max_kv", "var_avg_spare_kv", "var_avg_spare_queue", "mod_avg_spare_kv", "mod_avg_spare_queue"):
        assert _bit_equal(rd[k], o[k]), k
