"""wva_grid_update: the resident replica grid brought up to date after wva_update_servers by re-evaluating only the
servers whose load changed, held bit for bit, on every array wva_grid_fetch returns, to a second context's
load_system(new system) + grid_run and, on small fleets, to the oracle."""
import re
import threading

import numpy as np
import pytest

from tests.test_grid_edges import OVERFLOW_R, OVERFLOW_ROWS, _alpha_system, _classify_levels
from tests.test_recalculate import CYCLE, _bits, _expected_counts, _fleet, _next_cycle, _same

LOAD = ("srv_arrival", "srv_in_tokens", "srv_out_tokens")
GRID = ("ok", "ttft", "itl", "rho", "tput")
COUNTERS = ("chain_solves", "chain_states", "overflow_pairs", "certify_fallbacks")
OPT_GRID_DEFER = 6


def _update(eng, d):
    eng.update_servers(*(d[k] for k in CYCLE))


def _expected_regrid(*specs):
    """servers whose load changed bitwise in at least one of the updates through specs[1:], starting from specs[0]"""
    changed = False
    for a, b in zip(specs, specs[1:]):
        for k in LOAD:
            changed = changed | (_bits(a[k]).reshape(a[k].size, -1) != _bits(b[k]).reshape(b[k].size, -1)).any(axis=1)
    return int(np.sum(changed))


def _assert_grid_equal(got, want, full):
    for k in ("frontier",) + (GRID if full else ()):
        assert _same(got[k], want[k]), (k, np.argwhere(got[k] != want[k])[:5])


def _matches_full_run(inc, ref, n, R, full, oracle=None):
    """inc's resident grid against ref after load_system(n) + grid_run(R, full), and against the oracle"""
    got = inc.grid_fetch(full)
    ref.load_system(n)
    ref.grid_run(R, full=full)
    _assert_grid_equal(got, ref.grid_fetch(full), full)
    if oracle is not None:
        _assert_grid_equal(got, oracle.analyze_grid(n, R, full=full), full)
    return got


def _reserved(err):
    """(deferral slots reserved, deferral list capacity) of each grid pass the debug output reports"""
    return [(int(a), int(b)) for a, b in re.findall(r"deferral reserved (\d+) of capacity (\d+)", err)]


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


FRACS = (0.0, 0.001, 0.01, 0.1, 0.5, 1.0, 0.0, 0.01, 0.001, 0.5, 0.1, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("full", [True, False])
def test_chained_cycles_match_grid_run_and_oracle(pkg, inc, ref, oracle, full):
    """12 cycles at 0-100 % changed loads, current-allocation-only changes mixed in (one cycle has only those)"""
    R = 32
    d = _fleet(pkg, 600, 8, R, stream=61)
    inc.load_system(d)
    inc.grid_run(R, full=full)
    g = np.random.default_rng(11)
    for cycle, frac in enumerate(FRACS):
        n = _next_cycle(d, g, frac, 0.0 if cycle == 8 else 0.03)
        _update(inc, n)
        assert inc.grid_update() == _expected_regrid(d, n), cycle
        _matches_full_run(inc, ref, n, R, full, oracle)
        d = n


@pytest.mark.gpu
@pytest.mark.parametrize("full", [True, False])
def test_chained_cycles_on_a_fleet_that_defers(pkg, inc, ref, capfd, monkeypatch, full):
    """3000 servers x 16 accelerators: the deferred pass runs by default where the changed servers have 20 000 pairs or
    more (50 and 100 %), and not below"""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    R, A = 32, 16
    d = _fleet(pkg, 3000, A, R, stream=67)
    inc.load_system(d)
    inc.grid_run(R, full=full)
    g = np.random.default_rng(13)
    for cycle, frac in enumerate(FRACS):
        n = _next_cycle(d, g, frac, 0.0 if cycle == 8 else 0.03)
        _update(inc, n)
        capfd.readouterr()
        D = inc.grid_update()
        passes = _reserved(capfd.readouterr().err)
        assert D == _expected_regrid(d, n), cycle
        if D == 0:
            assert passes == [] and all(inc.timing()[k] == 0 for k in COUNTERS)
        else:
            assert len(passes) == 1 and (passes[0][1] > 0) == (D * A >= 20000), (cycle, D, passes)
        _matches_full_run(inc, ref, n, R, full)
        d = n


@pytest.mark.gpu
@pytest.mark.parametrize("full", [True, False])
def test_deferred_and_overflow_passes_inside_an_update(pkg, inc, ref, oracle, capfd, monkeypatch, full):
    """Forced deferral on four changed servers whose new loads put levels of the main and of the deferred pass past
    float64 (test_grid_edges: test_overflow_system_reaches_every_chain_kind); a fifth, unchanged server overflows in
    the resident grid only."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    new = _alpha_system(pkg, OVERFLOW_ROWS + [(1024, 160000.0), (64, 500.0)])
    old = dict(new)
    old["srv_arrival"] = new["srv_arrival"].copy()
    old["srv_arrival"][:4] = np.float32(60.0 * 50.0)          # light loads: nothing overflows before the update
    changed = {0, 1, 2, 3}
    n_ovf = sum(k in ("term", "sum") for s, *_, k in _classify_levels(new, OVERFLOW_R) if s in changed)
    assert n_ovf > 0
    inc.set_option(OPT_GRID_DEFER, 2)
    ref.set_option(OPT_GRID_DEFER, 2)
    inc.load_system(old)
    inc.grid_run(OVERFLOW_R, full=full)
    _update(inc, new)
    capfd.readouterr()
    assert inc.grid_update() == 4
    passes = _reserved(capfd.readouterr().err)
    assert len(passes) == 1 and passes[0][0] > 0, passes
    assert inc.timing()["overflow_pairs"] == n_ovf
    _matches_full_run(inc, ref, new, OVERFLOW_R, full, oracle)


@pytest.mark.gpu
@pytest.mark.parametrize("full", [True, False])
def test_every_server_changed(pkg, inc, ref, oracle, full):
    """every load of the block changed: the update evaluates the resident rows in place, with a grid_run's counters"""
    R = 16
    d = _fleet(pkg, 300, 6, R, stream=97)
    inc.load_system(d)
    inc.grid_run(R, full=full)
    n = dict(d)
    n["srv_arrival"] = (d["srv_arrival"] + np.float32(0.25)).astype(np.float32)
    _update(inc, n)
    assert inc.grid_update() == 300
    got = inc.timing()
    _matches_full_run(inc, ref, n, R, full, oracle)
    want = ref.timing()
    assert all(got[k] == want[k] for k in COUNTERS), ({k: got[k] for k in COUNTERS}, {k: want[k] for k in COUNTERS})


@pytest.mark.gpu
def test_edge_cases(pkg, inc, ref, oracle):
    R = 16
    d = _fleet(pkg, 400, 6, R, stream=71)
    inc.load_system(d)
    inc.grid_run(R, full=True)
    before = inc.grid_fetch()
    # nothing marked, with and without an update
    for do_update in (False, True):
        if do_update:
            _update(inc, d)
        assert inc.grid_update() == 0
        assert all(inc.timing()[k] == 0 for k in COUNTERS)
        _assert_grid_equal(inc.grid_fetch(), before, True)
    # a current-allocation-only change, cur_acc moves on keepAccelerator servers among them: nothing re-evaluated
    g = np.random.default_rng(17)
    alloc = _next_cycle(d, g, 0.0, 0.5)
    keep = d["srv_keep_acc"] != 0
    assert (keep & (alloc["srv_cur_acc"] != d["srv_cur_acc"])).any()
    _update(inc, alloc)
    assert inc.grid_update() == 0
    _assert_grid_equal(inc.grid_fetch(), before, True)
    # -0.0 <-> 0.0 is a change, with the same bits
    zero = np.flatnonzero(alloc["srv_arrival"] == 0)
    assert zero.size > 0
    n = dict(alloc)
    n["srv_arrival"] = alloc["srv_arrival"].copy()
    n["srv_arrival"][zero] = np.float32(-0.0)
    _update(inc, n)
    assert inc.grid_update() == zero.size
    _assert_grid_equal(inc.grid_fetch(), before, True)
    # loads to and from zero, out_tokens to 0 and back
    busy = np.flatnonzero(n["srv_arrival"] > 0)
    m1 = dict(n)
    for k in LOAD:
        m1[k] = n[k].copy()
    m1["srv_arrival"][busy[:15]] = 0.0
    m1["srv_arrival"][zero] = np.float32(125.5)
    m1["srv_out_tokens"][busy[15:30]] = 0
    _update(inc, m1)
    assert inc.grid_update() == 30 + zero.size
    _matches_full_run(inc, ref, m1, R, True, oracle)
    m2 = dict(m1)
    for k in LOAD:
        m2[k] = m1[k].copy()
    m2["srv_arrival"][zero] = 0.0
    m2["srv_out_tokens"][busy[15:30]] = n["srv_out_tokens"][busy[15:30]]
    _update(inc, m2)
    assert inc.grid_update() == 15 + zero.size
    _matches_full_run(inc, ref, m2, R, True, oracle)
    # two updates composed before one grid update (a load changed and changed back counts as changed)
    c1 = _next_cycle(m2, g, 0.1, 0.1)
    c2 = _next_cycle(c1, g, 0.05, 0.05)
    back = np.flatnonzero(c1["srv_arrival"] != m2["srv_arrival"])[:5]
    c2["srv_arrival"][back] = m2["srv_arrival"][back]
    _update(inc, c1)
    _update(inc, c2)
    got = inc.grid_update()
    assert got == _expected_regrid(m2, c1, c2) and got > _expected_regrid(m2, c2)
    _matches_full_run(inc, ref, c2, R, True)
    # update -> grid_run -> grid_update: the run consumed the marks
    c3 = _next_cycle(c2, g, 0.2, 0.1)
    _update(inc, c3)
    inc.grid_run(R, full=True)
    assert inc.grid_update() == 0
    _matches_full_run(inc, ref, c3, R, True)


@pytest.mark.gpu
@pytest.mark.parametrize("grid_first", [False, True])
def test_grid_and_sizing_marks_are_apart(pkg, inc, ref, grid_first):
    """update -> recalculate -> grid update and update -> grid update -> recalculate: neither call consumes the other's
    marks, and a calculate leaves the grid marks too"""
    R = 16
    d = _fleet(pkg, 500, 8, R, stream=73)
    inc.load_system(d)
    inc.calculate()
    inc.grid_run(R, full=True)
    g = np.random.default_rng(19)
    for frac in (0.05, 0.3):
        n = _next_cycle(d, g, frac, 0.05)
        _update(inc, n)
        if grid_first:
            assert inc.grid_update() == _expected_regrid(d, n)
            assert inc.recalculate() == _expected_counts(d, n)
        else:
            assert inc.recalculate() == _expected_counts(d, n)
            assert inc.grid_update() == _expected_regrid(d, n)
        ref.load_system(n)
        ref.calculate()
        want = ref.candidates()
        got = inc.candidates()
        for k in ("state", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate"):
            assert _same(got[k], want[k]), k
        _matches_full_run(inc, ref, n, R, True)
        d = n
    n = _next_cycle(d, g, 0.1, 0.0)
    _update(inc, n)
    inc.calculate()
    assert inc.grid_update() == _expected_regrid(d, n) > 0
    _matches_full_run(inc, ref, n, R, True)


@pytest.mark.gpu
def test_error_and_state_rules(pkg, inc, ref):
    R = 8
    d = pkg.synth.queue_system(6, 2, 64, stream=79, R=R, zero_load_frac=0.0, infeasible_frac=0.0)
    assert d["srv_model"][2] >= 0 and d["perf_present"][d["srv_model"][2]].any() and d["srv_arrival"][2] > 0
    d["srv_max_batch"][:] = 0
    d["perf_max_batch"][:] = 64
    d["perf_at_tokens"][:] = 200
    d["srv_out_tokens"][:] = 100                                # N = 64 * 200 / out_tokens = 128
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.grid_update()                                       # nothing loaded
    inc.load_system(d)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.grid_update()                                       # no grid run
    inc.grid_run(R, full=True)
    assert inc.grid_update() == 0
    assert all(inc.timing()[k] == 0 for k in COUNTERS)
    # another system loaded: refused until the next grid_run
    other = _fleet(pkg, 50, 3, R, stream=83)
    inc.load_system(other)
    _update(inc, other)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.grid_update()
    inc.grid_run(R, full=False)
    assert inc.grid_update() == 0
    # a failed grid update (out_tokens 1 gives N = 12 800, above the batch size limit) is refused after
    inc.load_system(d)
    inc.grid_run(R, full=True)
    bad = dict(d)
    bad["srv_out_tokens"] = d["srv_out_tokens"].copy()
    bad["srv_out_tokens"][2] = 1
    _update(inc, bad)
    with pytest.raises(pkg.WvaError, match="10188"):
        inc.grid_update()
    _update(inc, d)
    with pytest.raises(pkg.WvaError, match="call order"):
        inc.grid_update()
    inc.grid_run(R, full=True)
    assert inc.grid_update() == 0
    _matches_full_run(inc, ref, d, R, True)


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.gpu
@pytest.mark.skipif("_n_gpus() < 2", reason="needs two GPUs")
def test_two_ranks_update_their_blocks(pkg, ref):
    R = 16
    d = _fleet(pkg, 2001, 6, R, stream=89)
    n = _next_cycle(d, np.random.default_rng(23), 0.2, 0.1)
    ref.load_system(n)
    ref.grid_run(R, full=True)
    one = ref.grid_fetch()
    uid = pkg.comm_unique_id()
    res, errs, counts = [None, None], [], [None, None]

    def rank(r):
        try:
            with pkg.Engine(device=r) as e:
                e.comm_init(2, r, uid)
                e.load_system(d)
                e.grid_run(R, full=True)
                _update(e, n)
                counts[r] = e.grid_update()
                res[r] = (e.lo, e.hi, e.grid_fetch())
        except Exception as ex:   # noqa: BLE001  (reported by the main thread)
            errs.append(ex)

    th = [threading.Thread(target=rank, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    assert counts[0] + counts[1] == _expected_regrid(d, n)
    for lo, hi, got in res:
        _assert_grid_equal(got, {k: v[lo:hi] for k, v in one.items()}, True)
