"""wva_update_server_set: the server set of a loaded system replaced in place (servers added, removed and re-specified)
and only the servers that changed re-sized and re-gridded, held bit for bit to a second context's load_system(new) +
calculate (+ grid_run) and to the oracle; server_set_prev, the host rule that decides when a caller may take the path.

Every fleet is a subset of a "universe" of servers whose index is their name order, so that a cycle's system is a set
of universe rows plus column edits and `prev` follows from the universe indices."""
import copy
import re
import threading

import numpy as np
import pytest

from tests import ref_scenarios
from tests.test_grid_edges import OVERFLOW_R, OVERFLOW_ROWS, _alpha_system
from tests.test_recalculate import CAND, CYCLE, _assert_cand_equal, _bits, _fleet, _marks, _next_cycle, _solutions_equal

SRV = ("srv_model", "srv_priority", "srv_min_replicas", "srv_max_batch", "srv_keep_acc", "srv_target_present",
       "srv_slo_ttft", "srv_slo_itl", "srv_slo_tps") + CYCLE
LOAD = ("srv_arrival", "srv_in_tokens", "srv_out_tokens")
GRIDDED = LOAD + ("srv_model", "srv_max_batch", "srv_target_present", "srv_slo_ttft", "srv_slo_itl", "srv_slo_tps")
GRID = ("ok", "ttft", "itl", "rho", "tput")
OPT_FORCE_LANE_SIZER, OPT_GRID_DEFER = 1, 6


def _subset(u, ids):
    """the system of universe servers `ids` (ascending)"""
    d = dict(u)
    d["n_servers"] = len(ids)
    for k in SRV:
        d[k] = u[k][ids].copy()
    return d


def _prev(old_ids, new_ids):
    pos = {int(g): i for i, g in enumerate(old_ids)}
    return np.array([pos.get(int(g), -1) for g in new_ids], np.int32)


def _differs(a, b):
    return (_bits(a).reshape(a.size, -1) != _bits(b).reshape(b.size, -1)).any(axis=1)


class Marks:
    """the mark table of include/wva_b200.h, kept on the host: (re-size, current allocation changed, grid) per server of
    the resident set, accumulated from update to update until a recalculate / grid update consumes them"""

    def __init__(self, S):
        self.resize, self.alloc, self.grid = (np.zeros(S, bool) for _ in range(3))

    def update_servers(self, old, new):
        r, a = _marks(old, new)
        self.resize |= r
        self.alloc |= a
        for k in LOAD:
            self.grid |= _differs(old[k], new[k])

    def server_set(self, old, new, prev):
        kept, p = prev >= 0, prev[prev >= 0]
        diff = {}
        for k in SRV:
            diff[k] = np.ones(prev.size, bool)
            diff[k][kept] = _differs(old[k][p], new[k][kept])
        grid = np.logical_or.reduce([diff[k] for k in GRIDDED])
        keep_old = np.ones(prev.size, bool)
        keep_old[kept] = old["srv_keep_acc"][p] != 0
        moved = diff["srv_cur_acc"]
        resize = grid | diff["srv_min_replicas"] | diff["srv_keep_acc"] | (moved & (keep_old | (new["srv_keep_acc"] != 0)))
        alloc = moved | diff["srv_cur_replicas"] | diff["srv_cur_cost"]
        carry = lambda m: np.where(kept, m[np.maximum(prev, 0)] if m.size else False, False)
        self.resize = carry(self.resize) | resize
        self.alloc = carry(self.alloc) | alloc
        self.grid = carry(self.grid) | grid

    def recalculated(self):
        got = int(self.resize.sum()), int((self.alloc & ~self.resize).sum())
        self.resize[:], self.alloc[:] = False, False
        return got

    def regridded(self):
        got = int(self.grid.sum())
        self.grid[:] = False
        return got


def _edit(u, g, frac, ids):
    """a copy of universe u with every kind of server column edit on `frac` of the servers `ids`: SLOs, min replicas,
    max batch, keepAccelerator, target present, model (to -1 among them), priority, loads and current allocations"""
    n = dict(u)
    for k in SRV:
        n[k] = u[k].copy()
    A, M = int(u["n_acc"]), int(u["n_models"])
    pick = lambda: g.permutation(ids)[: max(1, int(round(frac * len(ids))))] if frac > 0 else np.zeros(0, int)
    i = pick(); n["srv_slo_itl"][i] = np.round(n["srv_slo_itl"][i] * np.float32(1.25) + 1, 1).astype(np.float32)
    i = pick(); n["srv_slo_ttft"][i] = np.round(n["srv_slo_ttft"][i] * np.float32(0.8) + 5, 1).astype(np.float32)
    i = pick(); n["srv_min_replicas"][i] = g.integers(0, 4, i.size)
    i = pick(); n["srv_max_batch"][i] = np.where(g.random(i.size) < 0.5, 0, g.integers(8, 64, i.size))
    i = pick(); n["srv_keep_acc"][i] ^= 1
    i = pick(); n["srv_target_present"][i] ^= 1
    i = pick(); n["srv_model"][i] = np.where(g.random(i.size) < 0.3, -1, g.integers(0, M, i.size))
    i = pick(); n["srv_priority"][i] = g.integers(1, 4, i.size)
    i = pick(); n["srv_arrival"][i] = np.round(n["srv_arrival"][i] * np.float32(1.3) + 0.5, 2).astype(np.float32)
    i = pick(); n["srv_out_tokens"][i] = g.integers(8, 512, i.size)
    i = pick()
    acc = g.integers(-2, A, i.size).astype(np.int32)
    n["srv_cur_acc"][i] = acc
    n["srv_cur_replicas"][i] = np.where(acc >= 0, g.integers(1, 6, i.size), 0)
    n["srv_cur_cost"][i] = np.where(acc >= 0, g.uniform(10, 500, i.size), 0).astype(np.float32)
    return n


def _churn(ids, U, g, frac, where):
    """`ids` with round(frac * len) servers removed and as many added from the rest of the universe [0, U), at the
    front (lowest indices), at the back (highest) or interleaved (at random)"""
    k = int(round(frac * len(ids)))
    if k == 0:
        return ids.copy()
    out = np.setdiff1d(np.arange(U), ids)
    if where == "front":
        gone, new = ids[:k], out[:k]
    elif where == "back":
        gone, new = ids[-k:], out[-k:]
    else:
        gone, new = g.choice(ids, k, replace=False), g.choice(out, k, replace=False)
    return np.union1d(np.setdiff1d(ids, gone), new)


def _set_update(eng, marks, old, new, prev):
    marks.server_set(old, new, prev)
    eng.update_server_set(prev, new)


def _calc_equal(inc, full, n):
    full.load_system(n)
    full.calculate()
    got = inc.candidates()
    _assert_cand_equal(got, full.candidates())
    return got


def _grid_equal(inc, ref, n, R, full, oracle=None):
    got = inc.grid_fetch(full)
    ref.load_system(n)
    ref.grid_run(R, full=full)
    want = ref.grid_fetch(full)
    for k in ("frontier",) + (GRID if full else ()):
        assert np.array_equal(_bits(got[k]), _bits(want[k])), (k, np.argwhere(got[k] != want[k])[:5])
    if oracle is not None:
        o = oracle.analyze_grid(n, R, full=full)
        for k in ("frontier",) + (GRID if full else ()):
            assert np.array_equal(_bits(got[k]), _bits(o[k])), k


@pytest.fixture
def inc(pkg):
    eng = pkg.Engine(device=0)
    yield eng
    eng.close()


@pytest.fixture
def ref(pkg):
    eng = pkg.Engine(device=0)
    yield eng
    eng.close()


# churn share, where, share of column edits, an update_servers call before the set update (marks carried across it)
CYCLES = ((0.0, "front", 0.0, False), (0.001, "front", 0.01, False), (0.01, "back", 0.05, True),
          (0.1, "mixed", 0.02, False), (0.5, "mixed", 0.1, True), (0.01, "front", 0.0, False),
          (0.1, "back", 0.3, False), (0.001, "mixed", 0.01, True), (0.5, "front", 0.05, False),
          (0.0, "back", 0.05, True), (0.1, "mixed", 0.0, False), (0.01, "mixed", 0.2, True))


@pytest.mark.gpu
def test_chained_cycles_match_calculate_and_oracle(pkg, engine, inc, oracle):
    U, S = 6000, 3000
    u = _fleet(pkg, U, 16, 64, stream=101)
    g = np.random.default_rng(29)
    ids = np.arange(1500, 1500 + S)
    d = _subset(u, ids)
    inc.load_system(d)
    inc.calculate()
    marks = Marks(S)
    for cycle, (churn, where, edits, between) in enumerate(CYCLES):
        if between:                                   # loads and allocations first, on the old set
            mid = _next_cycle(d, g, 0.05, 0.05)
            marks.update_servers(d, mid)
            inc.update_servers(*(mid[k] for k in CYCLE))
            u = dict(u)
            for k in CYCLE:                           # the universe follows
                u[k] = u[k].copy()
                u[k][ids] = mid[k]
            d = mid
        new_ids = _churn(ids, U, g, churn, where)
        u = _edit(u, g, edits, new_ids)
        n = _subset(u, new_ids)
        _set_update(inc, marks, d, n, _prev(ids, new_ids))
        assert inc.S == len(new_ids)
        assert inc.recalculate() == marks.recalculated(), cycle
        got = _calc_equal(inc, engine, n)
        if cycle in (2, 7):
            _assert_cand_equal(got, oracle.calculate(n))
        _solutions_equal(pkg, inc, engine, n, None)
        ids, d = new_ids, n


@pytest.mark.gpu
def test_counts_and_a_priority_only_cycle(pkg, engine, inc):
    """n_resized / n_revalued / n_regridded against the host mark table, one column kind at a time; a priority-only
    cycle re-sizes and re-grids nothing yet changes the limited solution"""
    U, R = 800, 16
    u = _fleet(pkg, U, 6, 32, stream=103)
    u["srv_priority"] = np.where(np.arange(U) % 2 == 0, 1, 3).astype(np.int32)
    ids = np.arange(0, U, 2)[:300]
    d = _subset(u, ids)
    inc.load_system(d)
    inc.calculate()
    inc.grid_run(R, full=False)
    marks = Marks(len(ids))
    g = np.random.default_rng(31)
    for k in SRV:
        n = dict(d)
        n[k] = d[k].copy()
        i = g.permutation(len(ids))[:25]
        if d[k].dtype == np.float32:
            n[k][i] = n[k][i] + np.float32(1.5)
        elif k in ("srv_keep_acc", "srv_target_present"):
            n[k][i] ^= 1
        elif k == "srv_cur_acc":
            n[k][i] = (n[k][i] + 3) % d["n_acc"]
        elif k == "srv_model":
            n[k][i] = -1
        else:
            n[k][i] = n[k][i] + 1
        _set_update(inc, marks, d, n, np.arange(len(ids), dtype=np.int32))
        want_rc, want_g = marks.recalculated(), marks.regridded()
        assert inc.recalculate() == want_rc, k
        assert inc.grid_update() == want_g, k
        assert (want_g > 0) == (k in GRIDDED), k
        if k == "srv_priority":
            assert want_rc == (0, 0)
        _calc_equal(inc, engine, n)
        d = n
    # priorities swapped across the fleet, nothing else: the limited solution follows them
    e = pkg.Engine(device=0)
    try:
        e.load_system(d)
        e.calculate()
        e.solve()
        cap = pkg.synth.limit_capacity(d, e.solution()["type_count"], 0.4)["type_count"]
        e.set_capacity(cap)
        e.set_optimizer(False, False, "PriorityRoundRobin")
        e.solve()
        before = e.solution()
    finally:
        e.close()
    n = dict(d)
    n["srv_priority"] = (4 - d["srv_priority"]).astype(np.int32)
    inc.update_server_set(np.arange(len(ids), dtype=np.int32), n)
    assert inc.recalculate() == (0, 0) and inc.grid_update() == 0
    inc.set_capacity(cap)
    inc.set_optimizer(False, False, "PriorityRoundRobin")
    inc.solve()
    after = inc.solution()
    assert not all(np.array_equal(after[k], before[k]) for k in ("state", "acc", "num_replicas"))
    _calc_equal(inc, engine, n)
    _solutions_equal(pkg, inc, engine, n, cap)


@pytest.mark.gpu
@pytest.mark.parametrize("full", [True, False])
def test_grid_follows_the_set(pkg, inc, ref, oracle, full):
    R, U = 32, 1200
    u = _fleet(pkg, U, 8, R, stream=107)
    g = np.random.default_rng(37)
    ids = np.arange(300, 900)
    d = _subset(u, ids)
    inc.load_system(d)
    inc.calculate()
    inc.grid_run(R, full=full)
    marks = Marks(len(ids))
    for cycle, (churn, where, edits, between) in enumerate(CYCLES[:8]):
        new_ids = _churn(ids, U, g, churn, where)
        u = _edit(u, g, edits, new_ids)
        n = _subset(u, new_ids)
        _set_update(inc, marks, d, n, _prev(ids, new_ids))
        if cycle % 2:
            assert inc.recalculate() == marks.recalculated()
        assert inc.grid_update() == marks.regridded(), cycle
        _grid_equal(inc, ref, n, R, full, oracle if cycle in (3, 6) else None)
        ids, d = new_ids, n


@pytest.mark.gpu
@pytest.mark.parametrize("full", [True, False])
def test_grid_on_a_fleet_that_defers(pkg, inc, ref, capfd, monkeypatch, full):
    """3000 x 16: the update's deferred pass runs where the changed servers have 20 000 pairs or more"""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    R, A, U = 32, 16, 4500
    u = _fleet(pkg, U, A, R, stream=109)
    g = np.random.default_rng(41)
    ids = np.arange(0, 3000)
    d = _subset(u, ids)
    inc.load_system(d)
    inc.grid_run(R, full=full)
    marks = Marks(len(ids))
    for churn, where in ((0.01, "front"), (0.5, "mixed"), (0.1, "back")):
        new_ids = _churn(ids, U, g, churn, where)
        n = _subset(u, new_ids)
        _set_update(inc, marks, d, n, _prev(ids, new_ids))
        capfd.readouterr()
        D = inc.grid_update()
        cap = [int(b) for b in re.findall(r"deferral reserved \d+ of capacity (\d+)", capfd.readouterr().err)]
        assert D == marks.regridded() and len(cap) == 1 and (cap[0] > 0) == (D * A >= 20000), (D, cap)
        _grid_equal(inc, ref, n, R, full)
        ids, d = new_ids, n


@pytest.mark.gpu
@pytest.mark.parametrize("full", [True, False])
def test_overflowing_servers_added_by_a_set_update(pkg, inc, ref, oracle, full):
    """servers whose levels overflow float64 arrive as new servers, into a grid with forced deferral"""
    u = _alpha_system(pkg, OVERFLOW_ROWS + [(64, 500.0), (128, 900.0)])
    inc.set_option(OPT_GRID_DEFER, 2)
    ref.set_option(OPT_GRID_DEFER, 2)
    old_ids, new_ids = np.array([4, 5]), np.arange(6)
    inc.load_system(_subset(u, old_ids))
    inc.calculate()
    inc.grid_run(OVERFLOW_R, full=full)
    n = _subset(u, new_ids)
    inc.update_server_set(_prev(old_ids, new_ids), n)
    assert inc.grid_update() == 4
    assert inc.timing()["overflow_pairs"] > 0
    _grid_equal(inc, ref, n, OVERFLOW_R, full, oracle)
    assert inc.recalculate() == (4, 0)
    _calc_equal(inc, ref, n)


@pytest.mark.gpu
def test_every_sizer_through_the_path(pkg, engine, inc, oracle):
    """the number of added servers picks the sizer of the recalculate: warp (<= 32 pairs per SM), lane, pool (> 640),
    and the lane sizer forced"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    A = 16
    U = 2 * sms * 700 // A + 200
    u = _fleet(pkg, U, A, 32, stream=113)
    ids = np.arange(0, U, 2)[:200]
    d = _subset(u, ids)
    inc.load_system(d)
    inc.calculate()
    seen = set()
    for D, force in ((sms * 16 // A, 0), (sms * 200 // A, 0), (sms * 700 // A, 0), (sms * 200 // A, 2)):
        inc.set_option(OPT_FORCE_LANE_SIZER, force)
        out = np.setdiff1d(np.arange(U), ids)
        new_ids = np.union1d(ids[: len(ids) // 2], out[np.linspace(0, out.size - 1, D).astype(int)])
        n = _subset(u, new_ids)
        inc.update_server_set(_prev(ids, new_ids), n)
        assert inc.recalculate()[0] == D
        seen.add(inc.timing()["sizer_kernel"])
        _calc_equal(inc, engine, n)
        ids, d = new_ids, n
    _assert_cand_equal(inc.candidates(), oracle.calculate(d))
    assert 1 in seen and 4 in seen and (2 in seen or 3 in seen), seen


@pytest.mark.gpu
def test_edges(pkg, engine, inc, ref):
    R, U = 16, 1000
    u = _fleet(pkg, U, 6, 32, stream=127)
    ids = np.arange(100, 400)
    d = _subset(u, ids)
    inc.load_system(d)
    inc.calculate()
    inc.grid_run(R, full=True)
    before = inc.candidates()
    # an identity prev with the same columns: nothing marked, nothing moved
    inc.update_server_set(np.arange(ids.size, dtype=np.int32), d)
    assert inc.recalculate() == (0, 0) and inc.grid_update() == 0
    _assert_cand_equal(inc.candidates(), before, CAND + ("n_solves",))
    # every server removed, then servers added into the empty system
    empty = _subset(u, ids[:0])
    inc.update_server_set(np.zeros(0, np.int32), empty)
    assert inc.S == 0 and inc.recalculate() == (0, 0) and inc.grid_update() == 0
    new_ids = np.arange(500, 560)
    n = _subset(u, new_ids)
    inc.update_server_set(np.full(new_ids.size, -1, np.int32), n)
    # before the recalculate / grid update: nil candidates and grid rows for the new servers; no solution yet
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.solution()
    c = inc.candidates()
    assert all(not np.any(c[k]) for k in CAND)
    gr = inc.grid_fetch(True)
    assert not gr["ok"].any() and not gr["frontier"].any()
    inc.solve()
    assert not inc.solution()["state"].any()
    assert inc.recalculate() == (new_ids.size, 0) and inc.grid_update() == new_ids.size
    _calc_equal(inc, engine, n)
    _grid_equal(inc, ref, n, R, True)
    # all servers new, and a set past the arenas' reserve (S doubling twice), then shrinking
    ids, d = new_ids, n
    for new_ids in (np.arange(600, 700), np.arange(0, 1000, 5), np.arange(0, 1000, 2), np.arange(3, 1000, 97)):
        n = _subset(u, new_ids)
        prev = _prev(ids, new_ids)
        inc.update_server_set(prev, n)
        inc.recalculate()
        inc.grid_update()
        _calc_equal(inc, engine, n)
        _grid_equal(inc, ref, n, R, True)
        ids, d = new_ids, n
    # a set update after set_candidates: recalculate is still refused
    inc.set_candidates(inc.candidates())
    new_ids = np.union1d(ids, [1, 2])
    n = _subset(u, new_ids)
    inc.update_server_set(_prev(ids, new_ids), n)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.recalculate()
    inc.calculate()
    assert inc.recalculate() == (0, 0)
    _calc_equal(inc, engine, n)


@pytest.mark.gpu
def test_error_rules_leave_the_context_unchanged(pkg, engine, inc):
    u = _fleet(pkg, 400, 4, 16, stream=131)
    ids = np.arange(50, 250)
    d = _subset(u, ids)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.update_server_set(np.zeros(0, np.int32), _subset(u, ids[:0]))   # nothing loaded
    inc.load_system(d)
    inc.calculate()
    mid = _next_cycle(d, np.random.default_rng(3), 0.1, 0.1)
    inc.update_servers(*(mid[k] for k in CYCLE))        # pending marks survive the refused calls
    new_ids = np.union1d(ids[10:], np.arange(300, 320))
    n = _subset(u, new_ids)
    good = _prev(ids, new_ids)
    bad = []
    p = good.copy(); p[5], p[6] = p[6], p[5]; bad.append((p, n))            # not increasing
    p = good.copy(); p[7] = p[6]; bad.append((p, n))                        # repeated
    p = good.copy(); p[0] = len(ids); bad.append((p, n))                    # out of range
    p = good.copy(); p[0] = -2; bad.append((p, n))
    m = dict(n); m["srv_model"] = n["srv_model"].copy(); m["srv_model"][3] = n["n_models"]; bad.append((good, m))
    m = dict(n); m["srv_cur_acc"] = n["srv_cur_acc"].copy(); m["srv_cur_acc"][3] = n["n_acc"]; bad.append((good, m))
    m = dict(n); m["srv_cur_acc"] = n["srv_cur_acc"].copy(); m["srv_cur_acc"][3] = -3; bad.append((good, m))
    for p, m in bad:
        with pytest.raises(pkg.WvaError, match="invalid argument"):
            inc.update_server_set(p, m)
    # a NULL column, through the C-ABI directly
    import ctypes as C
    st, keep = pkg._abi.make_system(n)
    st.srv_slo_tps = None
    rc = inc.lib.wva_update_server_set(inc.ctx, len(new_ids), good.ctypes.data, C.byref(st))
    assert rc == pkg._abi.WVA_ERR_ARG
    assert inc.S == len(ids)
    marks = Marks(len(ids))
    marks.update_servers(d, mid)
    assert inc.recalculate() == marks.recalculated()
    _calc_equal(inc, engine, mid)


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.gpu
@pytest.mark.skipif("_n_gpus() < 2", reason="needs two GPUs")
def test_two_ranks(pkg, engine):
    u = _fleet(pkg, 2400, 6, 32, stream=137)
    ids = np.arange(0, 2001)
    d = _subset(u, ids)
    n = _edit(u, np.random.default_rng(43), 0.1, ids)
    n = _subset(n, ids)
    want = engine.optimize(n)
    uid = pkg.comm_unique_id()
    res, errs = [None, None], []
    barrier = threading.Barrier(2)

    def rank(r):
        try:
            with pkg.Engine(device=r) as e:
                e.comm_init(2, r, uid)
                e.load_system(d)
                e.calculate()
                e.update_server_set(np.arange(len(ids), dtype=np.int32), n)
                e.recalculate()
                with pytest.raises(pkg.WvaError, match="call order"):
                    e.update_server_set(np.arange(1, len(ids), dtype=np.int32), _subset(u, ids[1:]))
                barrier.wait()
                e.solve()
                res[r] = e.solution()
        except Exception as ex:   # noqa: BLE001  (reported by the main thread)
            errs.append(ex)
            barrier.abort()

    th = [threading.Thread(target=rank, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for got in res:
        for k in ("state", "acc", "num_replicas", "cost", "value"):
            assert np.array_equal(_bits(got[k]), _bits(want[k])), k


# ---- CPU: server_set_prev and the binding -----------------------------------------------------------------------
def _flat(pkg, spec):
    return pkg.manager.flatten_spec(spec)


def test_server_set_prev_on_reference_specs(pkg):
    base = ref_scenarios.greedy_base()
    d0, i0 = _flat(pkg, base)
    # a membership change (server2 gone, server0 and server4 new) and column edits give a map by name
    s = copy.deepcopy(base)
    servers = [x for x in s["serverData"]["servers"] if x["name"] != "server2"]
    servers[0]["minNumReplicas"] = 3
    servers[1]["currentAlloc"]["load"]["arrivalRate"] = 99
    servers.append(dict(copy.deepcopy(servers[0]), name="server0"))
    servers.append(dict(copy.deepcopy(servers[0]), name="server4", **{"class": "low-priority"}))
    s["serverData"]["servers"] = servers
    d1, i1 = _flat(pkg, s)
    prev = pkg.manager.server_set_prev(i0, d0, i1, d1)
    assert i1.servers == ["server0", "server1", "server3", "server4"]
    assert prev.dtype == np.int32 and list(prev) == [-1, 0, 2, -1]
    # an SLO edit alone: the identity map
    t = copy.deepcopy(base)
    t["serviceClassData"]["serviceClasses"][0]["modelTargets"][0]["slo-itl"] = 123
    d2, i2 = _flat(pkg, t)
    assert list(pkg.manager.server_set_prev(i0, d0, i2, d2)) == [0, 1, 2]
    # an accelerator, a model or perf data changed: no map
    for edit in (lambda x: x["acceleratorData"]["accelerators"][0].update(cost=7.0),
                 lambda x: x["modelData"]["models"].append(dict(x["modelData"]["models"][0], name="llama-70b")),
                 lambda x: x["modelData"]["models"][1]["serviceParms"].update(alpha=9.0)):
        e = copy.deepcopy(s)
        edit(e)
        d3, i3 = _flat(pkg, e)
        assert pkg.manager.server_set_prev(i0, d0, i3, d3) is None


def test_binding_declares_the_header_prototype(pkg):
    import ctypes as C
    import os
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "wva_b200.h")).read()
    m = re.search(r"int32_t wva_update_server_set\(([^)]*)\);", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S))
    params = [p.strip().rsplit(" ", 1)[0].replace(" *", "*").strip() for p in m.group(1).split(",")]
    assert params == ["wva_ctx*", "int32_t", "const int32_t*", "const wva_system*"]
    L = pkg.engine.load_library()
    assert L.wva_update_server_set.argtypes == [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(pkg._abi.System)]
    assert "wva_update_server_set" in pkg.engine.EXPORTS
