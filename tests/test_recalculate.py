"""wva_update_servers + wva_recalculate: the per-cycle server columns (loads, current allocations) replaced in place and
only the servers they changed re-sized or re-valued, held bit for bit to a fresh load_system + calculate and to the
oracle; Manager.update's choice between that path and a full reload."""
import threading

import numpy as np
import pytest

CYCLE = ("srv_arrival", "srv_in_tokens", "srv_out_tokens", "srv_cur_acc", "srv_cur_replicas", "srv_cur_cost")
# every result field of a candidate; n_solves counts the chain solves the sizer spent, which depends on the sizer the
# dispatcher picks from the number of pairs it is handed and on how it batched them, so it is compared only where no
# pair was sized again
CAND = ("state", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate")
SOL = ("state", "acc", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate")
OPT_GREEDY_MODE = 5


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _assert_cand_equal(got, want, keys=CAND):
    for k in keys:
        assert _same(got[k], want[k]), (k, np.argwhere(np.asarray(got[k]) != np.asarray(want[k]))[:5])


def _marks(old, new):
    """the marks of one update, from a bitwise diff of the six columns: (re-size, current allocation changed) per server"""
    diff = {k: (_bits(old[k]).reshape(old[k].size, -1) != _bits(new[k]).reshape(new[k].size, -1)).any(axis=1)
            for k in CYCLE}
    resize = diff["srv_arrival"] | diff["srv_in_tokens"] | diff["srv_out_tokens"] | \
        (diff["srv_cur_acc"] & (old["srv_keep_acc"] != 0))
    return resize, diff["srv_cur_acc"] | diff["srv_cur_replicas"] | diff["srv_cur_cost"]


def _expected_counts(*specs):
    """(servers re-sized, servers re-valued only) after updates through specs[1:], starting from specs[0]"""
    resize = alloc = False
    for a, b in zip(specs, specs[1:]):
        r, v = _marks(a, b)
        resize, alloc = resize | r, alloc | v
    return int(np.sum(resize)), int(np.sum(alloc & ~resize))


def _fleet(pkg, S, A, N, stream):
    """queue_system with keepAccelerator servers, unknown models, live current allocations and every priority class"""
    d = pkg.synth.queue_system(S, A, N, stream=stream)
    g = np.random.default_rng(stream)
    d["srv_keep_acc"] = (g.random(S) < 0.3).astype(np.uint8)
    d["srv_model"] = np.where(g.random(S) < 0.03, -1, d["srv_model"]).astype(np.int32)
    cur = g.integers(-2, A, S).astype(np.int32)
    d["srv_cur_acc"] = cur
    d["srv_cur_replicas"] = np.where(cur >= 0, g.integers(1, 6, S), 0).astype(np.int32)
    d["srv_cur_cost"] = np.where(cur >= 0, d["acc_cost"][np.maximum(cur, 0)] * d["srv_cur_replicas"], 0).astype(np.float32)
    d["srv_arrival"] = np.round(d["srv_arrival"].astype(np.float64), 2).astype(np.float32)
    return d


def _next_cycle(d, g, load_frac, alloc_frac):
    """a copy of d whose loads changed on a `load_frac` share of the servers (arrival on the two-decimal grid, tokens
    now and then, a few idle) and whose current allocation alone changed on another `alloc_frac` share (keepAccelerator
    servers among them moving to -1 and -2)"""
    S, A = d["n_servers"], d["n_acc"]
    n = dict(d)
    for k in CYCLE:
        n[k] = d[k].copy()
    ld = g.permutation(S)[: int(round(load_frac * S))]
    arr = np.round(np.exp(g.uniform(np.log(0.5), np.log(60.0 * 100), ld.size)), 2)
    arr[g.random(ld.size) < 0.05] = 0.0
    n["srv_arrival"][ld] = arr.astype(np.float32)
    tok = ld[g.random(ld.size) < 0.2]
    n["srv_in_tokens"][tok] = g.integers(16, 2048, tok.size)
    n["srv_out_tokens"][tok] = g.integers(8, 512, tok.size)
    rest = np.setdiff1d(np.arange(S), ld)
    al = g.permutation(rest)[: int(round(alloc_frac * S))]
    acc = g.integers(-2, A, al.size).astype(np.int32)
    keep = al[d["srv_keep_acc"][al] != 0]
    acc[np.isin(al, keep[: keep.size // 3])] = -1
    acc[np.isin(al, keep[keep.size // 3: 2 * keep.size // 3])] = -2
    n["srv_cur_acc"][al] = acc
    n["srv_cur_replicas"][al] = np.where(acc >= 0, g.integers(1, 6, al.size), 0)
    n["srv_cur_cost"][al] = np.where(acc >= 0, g.uniform(10, 500, al.size), 0).astype(np.float32)
    return n


def _update(eng, d):
    eng.update_servers(*(d[k] for k in CYCLE))


def _recalc_equals_calculate(inc, full, n):
    """inc (just recalculated) against full after load_system(n) + calculate"""
    sizer = inc.timing()["sizer_kernel"]
    full.load_system(n)
    full.calculate()
    a = inc.candidates()
    _assert_cand_equal(a, full.candidates())
    return a, sizer


@pytest.fixture
def inc(pkg):
    eng = pkg.Engine(device=0)
    yield eng
    eng.close()


def _solutions_equal(pkg, inc, full, d, cap_of):
    """wva_solve on both contexts: unlimited, then limited under both greedy formulations"""
    for e in (inc, full):
        e.set_optimizer(True)
        e.solve()
    a, b = inc.solution(), full.solution()
    for k in SOL:
        assert _same(a[k], b[k]), k
    cap = pkg.synth.limit_capacity(d, a["type_count"], 0.6)["type_count"] if cap_of is None else cap_of
    for mode in (1, 2):
        for e in (inc, full):
            e.set_capacity(cap)
            e.set_optimizer(False, False, "PriorityRoundRobin")
            e.set_option(OPT_GREEDY_MODE, mode)
            e.solve()
        a, b = inc.solution(), full.solution()
        for k in SOL:
            assert _same(a[k], b[k]), (k, mode)
        assert np.array_equal(a["type_count"], b["type_count"])
    for e in (inc, full):
        e.set_option(OPT_GREEDY_MODE, 0)
        e.set_capacity(d["type_count"])
        e.set_optimizer(True)
    return cap


@pytest.mark.gpu
def test_chained_cycles_match_calculate_and_oracle(pkg, engine, inc, oracle):
    d = _fleet(pkg, 3000, 16, 64, stream=41)
    inc.load_system(d)
    inc.calculate()
    g = np.random.default_rng(7)
    cap = None
    for cycle, frac in enumerate((0.0, 0.001, 0.05, 0.3, 1.0, 0.0, 0.05, 0.001, 0.3, 0.0, 1.0, 0.05)):
        n = _next_cycle(d, g, frac, 0.0 if cycle == 9 else 0.03)
        _update(inc, n)
        got = inc.recalculate()
        assert got == _expected_counts(d, n), cycle
        c_inc, _ = _recalc_equals_calculate(inc, engine, n)
        _assert_cand_equal(c_inc, oracle.calculate(n))
        cap = _solutions_equal(pkg, inc, engine, n, cap)
        d = n


@pytest.mark.gpu
def test_every_sizer_through_the_gathered_view(pkg, engine, inc, oracle):
    """D picked on each side of the dispatcher's thresholds (pairs per SM): warp (<= 32), lane, pool (> 640)"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S, A = 8000, 16
    d = _fleet(pkg, S, A, 32, stream=43)
    inc.load_system(d)
    inc.calculate()
    seen = set()
    g = np.random.default_rng(9)
    for D in (sms * 16 // A, sms * 200 // A, min(S, sms * 700 // A)):
        n = dict(d)
        n["srv_arrival"] = d["srv_arrival"].copy()
        idx = g.permutation(S)[:D]
        n["srv_arrival"][idx] = np.round(n["srv_arrival"][idx] * 1.5 + 0.01, 2).astype(np.float32)
        _update(inc, n)
        assert inc.recalculate() == (D, 0)
        seen.add(_recalc_equals_calculate(inc, engine, n)[1])
        d = n
    _assert_cand_equal(inc.candidates(), oracle.calculate(d))
    assert 1 in seen and 4 in seen and (2 in seen or 3 in seen), seen


@pytest.mark.gpu
def test_float64_overflow_path_inside_recalculate(pkg, engine, inc, oracle):
    d = pkg.synth.queue_system(2, 2, 1024, stream=31)
    d["perf_alpha"][:] = 4.0
    d["perf_beta"][:] = 0.0
    d["perf_gamma"][:] = 0.0
    d["srv_in_tokens"][:] = 0
    d["srv_out_tokens"][:] = 16
    d["perf_at_tokens"][:] = 16
    d["srv_arrival"][:] = 60.0 * 20
    d["srv_slo_ttft"][:] = 5000.0
    d["srv_slo_itl"][:] = 0.0
    inc.load_system(d)
    inc.calculate()
    n = dict(d)
    n["srv_arrival"] = np.full(2, 60.0 * 2000, np.float32)
    _update(inc, n)
    assert inc.recalculate() == (2, 0)
    assert inc.timing()["overflow_pairs"] > 0
    _recalc_equals_calculate(inc, engine, n)
    _assert_cand_equal(inc.candidates(), oracle.calculate(n))


@pytest.mark.gpu
def test_edge_cases(pkg, engine, inc):
    d = _fleet(pkg, 500, 8, 32, stream=47)
    inc.load_system(d)
    inc.calculate()
    before = inc.candidates()
    # nothing changed, with and without an update
    for do_update in (False, True):
        if do_update:
            _update(inc, d)
        assert inc.recalculate() == (0, 0)
        t = inc.timing()
        assert t["chain_solves"] == 0 and t["sizer_kernel"] == 0 and t["overflow_pairs"] == 0
        _assert_cand_equal(inc.candidates(), before, CAND + ("n_solves",))
    # -0.0 <-> 0.0 is a change, with the same result
    zero = np.flatnonzero(d["srv_arrival"] == 0)
    assert zero.size > 0
    n = dict(d)
    n["srv_arrival"] = d["srv_arrival"].copy()
    n["srv_arrival"][zero] = np.float32(-0.0)
    _update(inc, n)
    assert inc.recalculate() == (zero.size, 0)
    _assert_cand_equal(inc.candidates(), before)
    # two updates between recalculates compose (one load changed and changed back counts as changed); loads to 0
    g = np.random.default_rng(3)
    m1 = _next_cycle(n, g, 0.1, 0.1)
    m1["srv_arrival"][:20] = 0.0
    m2 = _next_cycle(m1, g, 0.05, 0.05)
    back = np.flatnonzero(m1["srv_arrival"] != n["srv_arrival"])[:5]
    m2["srv_arrival"][back] = n["srv_arrival"][back]
    _update(inc, m1)
    _update(inc, m2)
    got = inc.recalculate()
    assert got == _expected_counts(n, m1, m2) and got[0] > _expected_counts(n, m2)[0]
    _recalc_equals_calculate(inc, engine, m2)


@pytest.mark.gpu
def test_error_and_state_rules(pkg, inc):
    d = _fleet(pkg, 200, 4, 16, stream=53)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.recalculate()
    with pytest.raises(pkg.WvaError, match="call order"):
        _update(inc, {k: d[k][:0] for k in CYCLE})   # nothing loaded: the binding's S is 0
    inc.load_system(d)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.recalculate()                           # after load_system, before calculate
    _update(inc, d)                                 # allowed; calculate voids the marks
    inc.calculate()
    assert inc.recalculate() == (0, 0)
    before = inc.candidates()
    bad = dict(d)
    bad["srv_arrival"] = d["srv_arrival"] + 1.0
    bad["srv_cur_acc"] = d["srv_cur_acc"].copy()
    bad["srv_cur_acc"][7] = d["n_acc"]
    with pytest.raises(pkg.WvaError, match="invalid argument"):
        _update(inc, bad)
    bad["srv_cur_acc"][7] = -3
    with pytest.raises(pkg.WvaError, match="invalid argument"):
        _update(inc, bad)
    assert inc.recalculate() == (0, 0)
    _assert_cand_equal(inc.candidates(), before, CAND + ("n_solves",))
    inc.set_candidates(before)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.recalculate()
    inc.calculate()
    assert inc.recalculate() == (0, 0)


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.gpu
@pytest.mark.skipif("_n_gpus() < 2", reason="needs two GPUs")
def test_two_ranks_update_their_blocks(pkg, engine):
    d = _fleet(pkg, 2001, 6, 32, stream=59)
    n = _next_cycle(d, np.random.default_rng(5), 0.2, 0.1)
    one = engine.optimize(n)
    cap = pkg.synth.limit_capacity(n, one["type_count"], 0.55)["type_count"]
    engine.set_capacity(cap)
    engine.set_optimizer(False)
    engine.solve()
    one_lim = engine.solution()
    uid = pkg.comm_unique_id()
    res, errs, counts = [None, None], [], [None, None]
    barrier = threading.Barrier(2)

    def rank(r):
        try:
            with pkg.Engine(device=r) as e:
                e.comm_init(2, r, uid)
                e.load_system(d)
                e.calculate()
                _update(e, n)
                counts[r] = e.recalculate()
                barrier.wait()
                e.solve()
                un = e.solution()
                e.set_capacity(cap)
                e.set_optimizer(False)
                e.solve()
                res[r] = (un, e.solution())
        except Exception as ex:   # noqa: BLE001  (reported by the main thread)
            errs.append(ex)
            barrier.abort()

    th = [threading.Thread(target=rank, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    rz, rv = _expected_counts(d, n)
    assert counts[0][0] + counts[1][0] == rz and counts[0][1] + counts[1][1] == rv
    for un, lim in res:
        for k in SOL:
            assert _same(un[k], one[k]) and _same(lim[k], one_lim[k]), k


# ---- Manager.update: the incremental path or a full reload (CPU, recording stub engine) -------------------------
class _Recorder:
    def __init__(self, S):
        self.calls, self.S = [], S

    def __getattr__(self, name):
        def rec(*a, **k):
            self.calls.append(name)
            if name in ("optimize", "solution"):
                z = np.zeros(self.S, np.int32)
                return {"state": z.astype(np.uint8), "acc": z, "num_replicas": z, "batch_size": z,
                        **{k: np.zeros(self.S, np.float32) for k in ("cost", "value", "itl", "ttft", "rho", "max_arrv_rate")},
                        "type_count": np.zeros(1, np.int64), "type_cost": np.zeros(1)}
            if name == "recalculate":
                return (0, 0)
        return rec


def _spec(arrival=30.0, cur_acc="H100", replicas=2, slo_itl=40.0):
    return {
        "acceleratorData": {"accelerators": [{"name": "A100", "type": "A100", "cost": 40.0, "multiplicity": 1},
                                             {"name": "H100", "type": "H100", "cost": 75.0, "multiplicity": 1}]},
        "capacityData": {"count": [{"type": "A100", "count": 8}, {"type": "H100", "count": 8}]},
        "modelData": {"models": [{"name": "m", "acc": a, "accCount": 1, "maxBatchSize": 64, "atTokens": 128,
                                  "serviceParms": {"alpha": 10.0, "beta": 0.1, "gamma": 0.001}} for a in ("A100", "H100")]},
        "serviceClassData": {"serviceClasses": [{"name": "Premium", "priority": 1,
                                                 "modelTargets": [{"model": "m", "slo-itl": slo_itl, "slo-ttft": 1000.0}]}]},
        "serverData": {"servers": [
            {"name": "s0", "class": "Premium", "model": "m", "keepAccelerator": True, "minNumReplicas": 1,
             "currentAlloc": {"accelerator": cur_acc, "numReplicas": replicas, "cost": 150.0,
                              "load": {"arrivalRate": arrival, "avgInTokens": 256, "avgOutTokens": 128}}},
            {"name": "s1", "class": "Premium", "model": "m", "minNumReplicas": 1,
             "currentAlloc": {"accelerator": "", "load": {"arrivalRate": 12.5, "avgInTokens": 64, "avgOutTokens": 32}}}]},
        "optimizerData": {"optimizer": {"unlimited": True}},
    }


def test_manager_update_picks_incremental_or_reload(pkg):
    full = ["load_system", "calculate", "solve", "solution"]
    incr = ["update_servers", "recalculate", "solve", "solution"]
    eng = _Recorder(2)
    m = pkg.Manager(eng, _spec())
    assert m.update(_spec(arrival=31.0)) == {"allocations": {}} and eng.calls == full   # nothing resident yet
    for spec, path in ((_spec(arrival=45.25), incr),                  # a load
                       (_spec(arrival=45.25, cur_acc="A100"), incr),  # a current allocation alone
                       (_spec(arrival=45.25, cur_acc="A100", replicas=3), incr),
                       (_spec(arrival=45.25, cur_acc="A100", replicas=3, slo_itl=50.0), full),   # an SLO
                       ({"system": _spec(arrival=0.0, cur_acc="A100", replicas=3, slo_itl=50.0)}, incr)):
        eng.calls.clear()
        m.update(spec)
        assert eng.calls == path, spec
    eng.calls.clear()
    m.optimize()
    m.update(_spec(arrival=0.0, cur_acc="", replicas=0, slo_itl=50.0))
    assert eng.calls == ["optimize"] + incr
    # the columns handed to update_servers are the new spec's, in the C-ABI's order
    seen = {}
    eng.update_servers = lambda *cols: seen.setdefault("cols", cols)
    m.update(_spec(arrival=7.5, cur_acc="H100", replicas=1, slo_itl=50.0))
    arr, tin, tout, acc, rep, cost = seen["cols"]
    assert arr.dtype == np.float32 and list(arr) == [7.5, 12.5] and list(acc) == [1, -1] and list(rep) == [1, 0]
    assert list(tin) == [256, 64] and list(tout) == [128, 32] and cost.dtype == np.float32
