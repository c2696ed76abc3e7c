"""wva_update_tables: the accelerator columns and perf tables of a loaded system replaced in place, and only the
(server, accelerator) pairs that read a changed row re-sized and re-gridded, held bit for bit to a second context's
load_system + calculate (+ grid_run) on the updated system and to the oracle; differs_only_in_tables, the host rule
that lets Manager.update take the path."""
import copy
import re
import threading

import numpy as np
import pytest

from tests import ref_scenarios
from tests.test_grid_edges import OVERFLOW_R, OVERFLOW_ROWS, _alpha_system
from tests.test_recalculate import CAND, SOL, _assert_cand_equal, _bits, _fleet, _next_cycle, _same, _solutions_equal
from tests.test_server_set import _prev, _subset

PERF = ("perf_alpha", "perf_beta", "perf_gamma", "perf_max_batch", "perf_at_tokens", "perf_acc_count", "perf_present")
ACC = ("acc_cost", "acc_multiplicity", "acc_type")
GRID = ("ok", "ttft", "itl", "rho", "tput")
OPT_FORCE_LANE_SIZER, OPT_GRID_DEFER = 1, 6
R = 24


def _differs(a, b):
    return (_bits(a).reshape(a.size, -1) != _bits(b).reshape(b.size, -1)).any(axis=1)


def _table_marks(old, new):
    """(sizing marks per perf row [M*A], cost marks per accelerator [A], grid marks per perf row) of one update"""
    d = {k: _differs(old[k], new[k]) for k in PERF}
    grid = np.logical_or.reduce([d[k] for k in PERF if k != "perf_acc_count"])
    return grid | d["perf_acc_count"], _differs(old["acc_cost"], new["acc_cost"]), grid


def _marked_pairs(sysd, rows, accs=None):
    """[S, A]: the pairs whose server's model is known and whose perf row (or accelerator) is marked"""
    A, model = int(sysd["n_acc"]), sysd["srv_model"]
    rows = rows.reshape(-1, A)
    hit = np.where(model[:, None] >= 0, rows[np.maximum(model, 0)], False)
    if accs is not None:
        hit = hit | ((model[:, None] >= 0) & accs[None, :])
    return hit


def _n_marked(old, new):
    size, cost, _ = _table_marks(old, new)
    return int(_marked_pairs(new, size, cost).sum())


def _tables(d, g, row_frac, acc_frac, fields=PERF + ACC):
    """a copy of d whose perf rows changed on a `row_frac` share (each field on its own share: alpha / beta / gamma
    scaled, max batch and at_tokens moved, acc_count, present toggled) and whose accelerator columns changed on an
    `acc_frac` share (cost, multiplicity, type, each on its own share)"""
    n = dict(d)
    for k in PERF + ACC:
        n[k] = d[k].copy()
    A, T = int(d["n_acc"]), int(d["n_types"])
    MA = d["perf_alpha"].size
    rows = lambda: g.permutation(MA)[: int(round(row_frac * MA))]
    accs = lambda: g.permutation(A)[: max(1, int(round(acc_frac * A)))] if acc_frac > 0 else np.zeros(0, int)
    flat = {k: n[k].reshape(-1) for k in PERF}
    for k in ("perf_alpha", "perf_beta", "perf_gamma"):
        if k in fields:
            i = rows()
            flat[k][i] = (flat[k][i] * g.uniform(0.7, 1.4, i.size)).astype(np.float32)
    if "perf_max_batch" in fields:
        i = rows()
        flat["perf_max_batch"][i] = np.maximum(1, flat["perf_max_batch"][i] + g.integers(-8, 9, i.size))
    if "perf_at_tokens" in fields:
        i = rows()
        flat["perf_at_tokens"][i] = np.maximum(1, flat["perf_at_tokens"][i] + g.integers(-16, 17, i.size))
    if "perf_acc_count" in fields:
        i = rows()
        flat["perf_acc_count"][i] = g.integers(1, 4, i.size)
    if "perf_present" in fields:
        i = rows()
        flat["perf_present"][i] ^= 1
    if "acc_cost" in fields:
        i = accs()
        n["acc_cost"][i] = np.round(n["acc_cost"][i] * np.float32(1.1) + 1, 2).astype(np.float32)
    if "acc_multiplicity" in fields:
        i = accs()
        n["acc_multiplicity"][i] = g.integers(1, 9, i.size)
    if "acc_type" in fields:
        i = accs()
        n["acc_type"][i] = g.integers(0, T, i.size)
    return n


def _full(eng, n, full_grid=None):
    eng.load_system(n)
    eng.calculate()
    if full_grid is not None:
        eng.grid_run(R, full_grid)


def _grid_equal(inc, ref, full_grid):
    ref.grid_run(R, full_grid)
    a, b = inc.grid_fetch(full_grid), ref.grid_fetch(full_grid)
    for k in ("frontier",) + (GRID if full_grid else ()):
        assert _same(a[k], b[k]), k


@pytest.fixture
def inc(pkg):
    eng = pkg.Engine(device=0)
    yield eng
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("full_grid", [True, False])
def test_chained_cycles_match_reload_and_oracle(pkg, engine, inc, oracle, full_grid):
    d = _fleet(pkg, 3000, 16, 64, stream=61)
    inc.load_system(d)
    inc.calculate()
    inc.grid_run(R, full_grid)
    g = np.random.default_rng(11)
    cap = None
    ids = np.arange(d["n_servers"])
    for cycle, (rf, af) in enumerate(((0.01, 0.0), (0.0, 0.1), (0.1, 0.2), (0.001, 0.0), (0.3, 0.5), (1.0, 1.0))):
        n = _tables(d, g, rf, af)
        if cycle in (1, 4):
            n = _next_cycle(n, g, 0.05, 0.03)
            inc.update_servers(*(n[k] for k in ("srv_arrival", "srv_in_tokens", "srv_out_tokens", "srv_cur_acc",
                                                "srv_cur_replicas", "srv_cur_cost")))
        if cycle == 2:   # a server set change between the table update and the recalculate
            keep = np.sort(g.permutation(ids.size)[: ids.size - 40])
            n2 = _subset(n, keep)
            assert inc.update_tables(n) == _n_marked(d, n)
            inc.update_server_set(_prev(np.arange(ids.size), keep), n2)
            n, ids = n2, ids[keep]
        else:
            assert inc.update_tables(n) == _n_marked(d, n), cycle
        inc.recalculate()
        inc.grid_update()
        _full(engine, n)
        _assert_cand_equal(inc.candidates(), engine.candidates())
        _grid_equal(inc, engine, full_grid)
        if cycle == 3:
            _assert_cand_equal(inc.candidates(), oracle.calculate(n))
        cap = _solutions_equal(pkg, inc, engine, n, cap)
        d = n


@pytest.mark.gpu
def test_n_marked_and_only_marked_pairs_resized(pkg, engine, inc):
    d = _fleet(pkg, 2000, 16, 32, stream=67)
    inc.load_system(d)
    inc.calculate()
    inc.grid_run(R, True)
    g = np.random.default_rng(13)
    # one accelerator's cost: every known-model pair on it, and no grid work
    n = dict(d)
    n["acc_cost"] = d["acc_cost"].copy()
    n["acc_cost"][5] += np.float32(3.0)
    before = inc.candidates()
    want = _marked_pairs(n, np.zeros(d["perf_alpha"].size, bool), np.arange(16) == 5)
    assert inc.update_tables(n) == int(want.sum()) > 0
    inc.recalculate()
    assert inc.timing()["chain_solves"] > 0
    got = inc.candidates()
    _full(engine, n)
    _assert_cand_equal(got, engine.candidates())
    for k in CAND + ("n_solves",):
        assert _same(got[k][~want], before[k][~want]), k
    assert inc.grid_update() == 0 and inc.timing()["chain_solves"] == 0
    _grid_equal(inc, engine, True)
    # alpha of one accelerator per model (a tuner's update): those pairs only, in the candidates and the grid
    d = n
    n = dict(d)
    n["perf_alpha"] = d["perf_alpha"].copy().reshape(-1, 16)
    col = g.integers(0, 16, n["perf_alpha"].shape[0])
    n["perf_alpha"][np.arange(col.size), col] *= np.float32(1.05)
    n["perf_alpha"] = n["perf_alpha"].reshape(d["perf_alpha"].shape)
    before = inc.candidates()
    size, cost, _ = _table_marks(d, n)
    want = _marked_pairs(n, size, cost)
    assert inc.update_tables(n) == int(want.sum())
    inc.recalculate()
    got = inc.candidates()
    _full(engine, n)
    _assert_cand_equal(got, engine.candidates())
    for k in CAND + ("n_solves",):
        assert _same(got[k][~want], before[k][~want]), k
    inc.grid_update()
    _grid_equal(inc, engine, True)


@pytest.mark.gpu
def test_every_sizer_through_the_pair_list(pkg, engine, inc, oracle):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S, A = 8000, 16
    d = _fleet(pkg, S, A, 32, stream=71)
    inc.load_system(d)
    inc.calculate()
    g = np.random.default_rng(17)
    seen = set()

    def step(n, expect=None):
        nonlocal d
        inc.update_tables(n)
        inc.recalculate()
        k = inc.timing()["sizer_kernel"]
        if expect is not None:
            assert k == expect
        seen.add(k)
        _full(engine, n)
        _assert_cand_equal(inc.candidates(), engine.candidates())
        d = n

    def alpha_rows(m_count):
        n = dict(d)
        n["perf_alpha"] = d["perf_alpha"].copy().reshape(-1, A)
        rows = g.permutation(n["perf_alpha"].shape[0])[:m_count]
        n["perf_alpha"][rows, :] *= np.float32(1.01)
        n["perf_alpha"] = n["perf_alpha"].reshape(d["perf_alpha"].shape)
        return n

    step(alpha_rows(max(1, sms * 16 // A)), 1)                # warp sizer: <= 32 pairs per SM
    for mode in range(1, 7):                                   # every forced lane-sizer mode (6: the pool)
        inc.set_option(OPT_FORCE_LANE_SIZER, mode)
        step(alpha_rows(sms * 4), 4 if mode == 6 else None)
    inc.set_option(OPT_FORCE_LANE_SIZER, 0)
    step(alpha_rows(min(S, sms * 760 // A)), 4)               # pool sizer: above 640 pairs per SM
    _assert_cand_equal(inc.candidates(), oracle.calculate(d))
    assert {1, 4} <= seen and (2 in seen or 3 in seen), seen


@pytest.mark.gpu
def test_float64_overflow_in_sizing_and_grid(pkg, engine, inc, oracle):
    d = _alpha_system(pkg, OVERFLOW_ROWS)
    small = dict(d)
    small["perf_alpha"] = np.full_like(d["perf_alpha"], 0.05)
    inc.load_system(small)
    inc.calculate()
    inc.grid_run(OVERFLOW_R, True)
    assert inc.update_tables(d) > 0
    inc.recalculate()
    assert inc.timing()["overflow_pairs"] > 0
    _full(engine, d)
    _assert_cand_equal(inc.candidates(), engine.candidates())
    _assert_cand_equal(inc.candidates(), oracle.calculate(d))
    inc.grid_update()
    assert inc.timing()["overflow_pairs"] > 0
    engine.grid_run(OVERFLOW_R, True)
    a, b = inc.grid_fetch(True), engine.grid_fetch(True)
    for k in ("frontier",) + GRID:
        assert _same(a[k], b[k]), k
    # the same with the deferred pass forced on the listed pairs
    for e in (inc, engine):
        e.set_option(OPT_GRID_DEFER, 2)
    try:
        inc.update_tables(small)
        inc.update_tables(d)            # a change and its revert: marked, the same result
        inc.grid_update()
        engine.grid_run(OVERFLOW_R, True)
        a, b = inc.grid_fetch(True), engine.grid_fetch(True)
        for k in ("frontier",) + GRID:
            assert _same(a[k], b[k]), k
    finally:
        for e in (inc, engine):
            e.set_option(OPT_GRID_DEFER, 0)


@pytest.mark.gpu
def test_mark_rules(pkg, engine, inc):
    d = _fleet(pkg, 600, 8, 32, stream=73)
    inc.load_system(d)
    inc.calculate()
    inc.grid_run(R, True)
    g = np.random.default_rng(19)
    base = inc.candidates()
    # marks accumulate over two updates; a change and its revert re-sizes with the same result
    n1 = _tables(d, g, 0.05, 0.0, ("perf_beta",))
    n2 = _tables(n1, g, 0.05, 0.0, ("perf_gamma",))
    back = dict(n2)
    back["perf_beta"] = d["perf_beta"]
    inc.update_tables(n1)
    inc.update_tables(back)
    inc.recalculate()
    want = _marked_pairs(back, _table_marks(d, n1)[0] | _table_marks(n1, back)[0])
    got = inc.candidates()
    _full(engine, back)
    _assert_cand_equal(got, engine.candidates())
    for k in CAND + ("n_solves",):
        assert _same(got[k][~want], base[k][~want]), k
    inc.grid_update()
    _grid_equal(inc, engine, True)
    d = back
    # -0.0 vs 0.0 is a change
    n = dict(d)
    n["perf_gamma"] = d["perf_gamma"].copy()
    n["perf_gamma"].reshape(-1)[:3] = 0.0
    inc.update_tables(n)
    inc.recalculate()
    d = n
    n = dict(d)
    n["perf_gamma"] = d["perf_gamma"].copy()
    n["perf_gamma"].reshape(-1)[:3] = np.float32(-0.0)
    assert inc.update_tables(n) == _n_marked(d, n) > 0
    inc.recalculate()
    assert inc.timing()["chain_solves"] > 0
    d = n
    # wva_calculate voids the sizing marks and leaves the grid marks; wva_grid_run voids the grid marks
    n = _tables(d, g, 0.1, 0.3)
    inc.update_tables(n)
    inc.calculate()
    assert inc.recalculate() == (0, 0) and inc.timing()["sizer_kernel"] == 0
    inc.grid_update()
    assert inc.timing()["chain_solves"] > 0
    _full(engine, n)
    _grid_equal(inc, engine, True)
    d = n
    n = _tables(d, g, 0.1, 0.0)
    inc.update_tables(n)
    inc.grid_run(R, True)
    inc.grid_update()
    assert inc.timing()["chain_solves"] == 0
    inc.recalculate()
    assert inc.timing()["sizer_kernel"] != 0
    _full(engine, n)
    _assert_cand_equal(inc.candidates(), engine.candidates())
    d = n
    # a model no server uses marks nothing
    unused = np.setdiff1d(np.arange(d["n_models"]), d["srv_model"])
    assert unused.size > 0
    n = dict(d)
    n["perf_alpha"] = d["perf_alpha"].copy().reshape(d["n_models"], -1)
    n["perf_alpha"][unused] *= np.float32(2.0)
    n["perf_alpha"] = n["perf_alpha"].reshape(d["perf_alpha"].shape)
    assert inc.update_tables(n) == 0
    assert inc.recalculate() == (0, 0) and inc.timing()["sizer_kernel"] == 0
    assert inc.grid_update() == 0 and inc.timing()["chain_solves"] == 0
    # multiplicities and types mark nothing; the allocators read them
    m = _tables(n, g, 0.0, 1.0, ("acc_multiplicity", "acc_type"))
    assert inc.update_tables(m) == 0
    inc.recalculate()
    assert inc.timing()["sizer_kernel"] == 0
    _full(engine, m)
    _assert_cand_equal(inc.candidates(), engine.candidates())
    _solutions_equal(pkg, inc, engine, m, None)


@pytest.mark.gpu
def test_error_and_state_rules(pkg, inc):
    import ctypes as C
    d = _fleet(pkg, 200, 4, 16, stream=79)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.update_tables(d)
    inc.load_system(d)
    inc.calculate()
    before = inc.candidates()
    bads = []
    b = dict(d); b["acc_type"] = d["acc_type"].copy(); b["acc_type"][1] = d["n_types"]; bads.append(b)
    b = dict(d); b["acc_type"] = d["acc_type"].copy(); b["acc_type"][0] = -1; bads.append(b)
    for k, v in (("perf_alpha", -1.0), ("perf_beta", np.nan), ("perf_gamma", np.inf)):
        b = dict(d); b[k] = d[k].copy(); b[k].reshape(-1)[2] = v; bads.append(b)
    b = dict(d); b["n_models"] = d["n_models"] + 1
    for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_max_batch", "perf_at_tokens", "perf_acc_count", "perf_present"):
        b[k] = np.concatenate([d[k].reshape(-1, 4), d[k].reshape(-1, 4)[:1]])
    bads.append(b)
    for b in bads:
        with pytest.raises(pkg.WvaError, match="invalid argument"):
            inc.update_tables(b)
    st, keep = pkg._abi.make_system({**d, "n_servers": 0, **{k: np.zeros(0, dt) for k, (dt, e) in
                                                              pkg._abi.SYSTEM_ARRAYS.items() if e == "S"}})
    st.perf_acc_count = None
    assert inc.lib.wva_update_tables(inc.ctx, C.byref(st), None) == 1
    # a present-off row may hold anything
    ok = dict(d)
    ok["perf_present"] = d["perf_present"].copy(); ok["perf_present"].reshape(-1)[3] = 0
    ok["perf_alpha"] = d["perf_alpha"].copy(); ok["perf_alpha"].reshape(-1)[3] = np.nan
    inc.update_tables(ok)
    inc.update_tables(d)
    assert inc.recalculate() == (0, 0)
    _assert_cand_equal(inc.candidates(), before)
    bad = bads[2]
    with pytest.raises(pkg.WvaError, match="invalid argument"):
        inc.update_tables(bad)
    assert inc.recalculate() == (0, 0) and inc.timing()["sizer_kernel"] == 0
    _assert_cand_equal(inc.candidates(), before, CAND + ("n_solves",))
    inc.set_candidates(before)
    inc.update_tables(_tables(d, np.random.default_rng(1), 0.2, 0.2))
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.recalculate()


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.gpu
@pytest.mark.skipif("_n_gpus() < 2", reason="needs two GPUs")
def test_two_ranks_equal_one_gpu(pkg, engine):
    d = _fleet(pkg, 2001, 6, 32, stream=83)
    n = _tables(d, np.random.default_rng(23), 0.1, 0.3)
    one = engine.optimize(n)
    uid = pkg.comm_unique_id()
    res, errs, marked = [None, None], [], [0, 0]
    barrier = threading.Barrier(2)

    def rank(r):
        try:
            with pkg.Engine(device=r) as e:
                e.comm_init(2, r, uid)
                e.load_system(d)
                e.calculate()
                marked[r] = e.update_tables(n)
                e.recalculate()
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
    assert marked[0] + marked[1] == _n_marked(d, n)
    for sol in res:
        for k in SOL:
            assert _same(sol[k], one[k]), k


# ---- CPU: the binding and the Manager's rule -------------------------------------------------------------------------
def test_binding_declares_the_header_prototype(pkg):
    import ctypes as C
    import os
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "wva_b200.h")).read()
    m = re.search(r"int32_t wva_update_tables\(([^)]*)\);", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S))
    params = [p.strip().rsplit(" ", 1)[0].replace(" *", "*").strip() for p in m.group(1).split(",")]
    assert params == ["wva_ctx*", "const wva_system*", "int64_t*"]
    L = pkg.engine.load_library()
    assert L.wva_update_tables.argtypes == [C.c_void_p, C.POINTER(pkg._abi.System), C.POINTER(C.c_int64)]
    assert "wva_update_tables" in pkg.engine.EXPORTS


def test_differs_only_in_tables_on_reference_specs(pkg):
    base = ref_scenarios.greedy_base()
    d0, _ = pkg.manager.flatten_spec(base)
    edits = {
        "cost": lambda x: x["acceleratorData"]["accelerators"][0].update(cost=7.0),
        "perf": lambda x: x["modelData"]["models"][1]["serviceParms"].update(alpha=9.0),
        "perf+load": lambda x: (x["modelData"]["models"][0]["serviceParms"].update(beta=0.5),
                                x["serverData"]["servers"][0]["currentAlloc"]["load"].update(arrivalRate=99)),
    }
    for name, edit in edits.items():
        e = copy.deepcopy(base)
        edit(e)
        d1, _ = pkg.manager.flatten_spec(e)
        assert pkg.manager.differs_only_in_tables(d0, d1), name
        assert not pkg.manager.differs_only_in_cycle_columns(d0, d1), name
    assert pkg.manager.differs_only_in_tables(d0, d0)
    # a new model, an SLO, a server or a capacity change is not a table update
    for edit in (lambda x: x["modelData"]["models"].append(dict(x["modelData"]["models"][0], name="llama-70b")),
                 lambda x: x["serviceClassData"]["serviceClasses"][0]["modelTargets"][0].update({"slo-itl": 123}),
                 lambda x: x["serverData"]["servers"].pop(),
                 lambda x: x["capacityData"]["count"][0].update(count=1)):
        e = copy.deepcopy(base)
        edit(e)
        d1, _ = pkg.manager.flatten_spec(e)
        assert not pkg.manager.differs_only_in_tables(d0, d1)


def test_manager_update_takes_the_table_path(pkg):
    from tests.test_recalculate import _Recorder
    base = ref_scenarios.greedy_base()
    S = len(base["serverData"]["servers"])
    eng = _Recorder(S)
    m = pkg.Manager(eng, base)
    m.optimize()
    e = copy.deepcopy(base)
    e["modelData"]["models"][1]["serviceParms"].update(alpha=9.0)
    eng.calls.clear()
    m.update(e)
    assert eng.calls == ["update_tables", "update_servers", "recalculate", "solve", "solution"]
    e2 = copy.deepcopy(e)
    e2["acceleratorData"]["accelerators"][0].update(cost=7.0)
    e2["modelData"]["models"].append(dict(e2["modelData"]["models"][0], name="llama-70b"))
    eng.calls.clear()
    m.update(e2)
    assert eng.calls == ["load_system", "calculate", "solve", "solution"]
