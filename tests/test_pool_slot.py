"""The pool sizer keeps a pair's state in global memory and moves only part of it per solve: the model and the hot block
(the bisection's fields) on every solve, the cold block (Size()'s tail and CreateAllocation) only when a step enters or
leaves the bisection, and never the chain's fields but its state count.  It claims new pairs a block of work items per
warp.  Forced pool sizer (set_option(1, 6)) on small systems whose pairs sit at different stages in one batch: every
candidate and n_solves bit-equal to the lane sizer (set_option(1, 2)), and every candidate bit-equal to the oracle (NaN
payloads aside), for a full calculate and for a recalculate over the pair list a table update marks."""
import numpy as np
import pytest

from tests.test_extreme_rates import RECIPES, _extreme, _same

CAND = ("state", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _assert_equal(got, want, keys, where):
    for k in keys:
        assert np.array_equal(_bits(got[k]), _bits(want[k])), (where, k, np.argwhere(np.asarray(got[k]) != np.asarray(want[k]))[:5])


def _assert_oracle(got, want):
    """bit for bit, but any NaN equals any NaN: the pair sized at lambda = inf (the "inf" recipe) reports NaN in
    max_arrv_rate, whose payload differs between the device and the x86 host (test_extreme_rates._same)"""
    for k in CAND:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        ok = _same(g, w) if g.dtype == np.float32 else np.array_equal(g, w)
        assert ok, ("oracle", k, np.argwhere(g != w)[:5])


def _slot_system(pkg, S=160, A=4, stream=71):
    """queue_system pairs (N = 64 and 32 mixed) with, on separate servers: TTFT targets below the bounded region (the
    search fails at xMax), both targets 0 (no search), a throughput target so small that the second Analyze rate
    underflows (alloc_replicas fails in SZ_FINAL1), no load, pairs without a perf row, keepAccelerator servers, service
    rates outside the (E1) divisor range (e1_ok == 0) and one pair whose chain overflows float64"""
    d = pkg.synth.queue_system(S, A, 64, stream=stream, zero_load_frac=0.0, infeasible_frac=0.0)
    rng = np.random.default_rng(stream)
    d["srv_max_batch"][:] = rng.choice(np.array([32, 64], np.int32), S)
    srv = np.arange(S)
    below = srv % 8 == 1
    d["srv_slo_ttft"][below] = 1e-6
    off = srv % 8 == 2
    d["srv_slo_ttft"][off] = 0.0
    d["srv_slo_itl"][off] = 0.0
    final1 = srv % 8 == 3
    d["srv_slo_tps"][final1] = 1e-38
    d["srv_min_replicas"][final1] = 1 << 30
    d["srv_arrival"][srv % 8 == 4] = 0.0
    d["perf_present"][(srv % 8 == 5)[:, None] & (np.arange(A) % 2 == 0)[None, :]] = 0
    keep = srv % 8 == 6
    d["srv_keep_acc"][keep] = 1
    d["srv_cur_acc"][keep] = srv[keep] % A
    d["srv_cur_replicas"][keep] = 1
    names = list(RECIPES)
    for k, s in enumerate(srv[srv % 8 == 7][:len(names)]):
        _extreme(d, [s], *RECIPES[names[k]])
    s = S - 1          # float64 overflow at the search's midpoints (test_recalculate's recipe)
    d["perf_alpha"][s] = 4.0
    d["perf_beta"][s] = 0.0
    d["perf_gamma"][s] = 0.0
    d["srv_in_tokens"][s] = 0
    d["srv_out_tokens"][s] = 16
    d["perf_at_tokens"][s] = 16
    d["srv_max_batch"][s] = 1024
    d["srv_arrival"][s] = 60.0 * 2000
    d["srv_slo_ttft"][s] = 5000.0
    d["srv_slo_itl"][s] = 0.0
    return d


def _calculate(engine, d, sizer):
    engine.set_option(1, sizer)
    try:
        engine.load_system(d)
        engine.calculate()
        return engine.candidates(), engine.timing()
    finally:
        engine.set_option(1, 0)


def test_slot_system_reaches_every_case(pkg, oracle):
    """the oracle's candidates show the cases the system is built for"""
    d = _slot_system(pkg)
    o = oracle.calculate(d)
    state = np.asarray(o["state"]).reshape(d["n_servers"], d["n_acc"])
    srv = np.arange(d["n_servers"])
    assert (state[srv % 8 == 1] == 0).any()                          # search failed
    assert (state[srv % 8 == 3] == 0).any()                          # alloc_replicas failed
    assert (state == 1).sum() > d["n_servers"]                       # and many sized pairs


@pytest.mark.gpu
@pytest.mark.parametrize("stream", [71, 72])
def test_pool_slot_matches_oracle_and_lane_sizer(pkg, engine, oracle, stream):
    d = _slot_system(pkg, stream=stream)
    g, t = _calculate(engine, d, 6)
    assert t["sizer_kernel"] == 4 and t["overflow_pairs"] > 0
    _assert_oracle(g, oracle.calculate(d))
    lane, _ = _calculate(engine, d, 2)
    _assert_equal(g, lane, CAND + ("n_solves",), "lane sizer")


@pytest.mark.gpu
def test_pool_slot_on_a_work_list(pkg, engine, oracle):
    """wva_update_tables marks the pairs of the models whose perf rows changed; recalculate sizes that list on the pool"""
    d = _slot_system(pkg, stream=73)
    eng = pkg.Engine(device=0)
    try:
        eng.set_option(1, 6)
        eng.load_system(d)
        eng.calculate()
        n = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
        rows = np.arange(0, d["n_models"], 3)
        n["perf_alpha"][rows] = n["perf_alpha"][rows] * np.float32(0.75)     # scaled down: some alphas are 3e38
        n["perf_gamma"][rows[::2]] = n["perf_gamma"][rows[::2]] * np.float32(0.5)
        assert eng.update_tables(n) > 0
        eng.recalculate()                           # the marked pairs, not servers: no server count
        t = eng.timing()
        assert t["sizer_kernel"] == 4 and t["chain_solves"] > 0
        got = eng.candidates()
    finally:
        eng.close()
    _assert_oracle(got, oracle.calculate(n))
    lane, _ = _calculate(engine, n, 2)
    _assert_equal(got, lane, CAND + ("n_solves",), "lane sizer")
