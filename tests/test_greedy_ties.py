"""Limited-capacity SolveGreedy on large tie groups and at the event sweep's size limit.

Every fixture is a system with SYNTHESIZED candidate tables (installed with wva_set_candidates; the oracle's greedy
takes the same tables), shaped so that the static-order event sweep (greedy_sweep.cuh) leaves its common path:

  wide       one priority class of 7 000 copies of one candidate row (and a second class behind it): the copies meet
             again as re-inserted leaders of one tau — more than GSW_DYN_CAP = 4 096 alive leaders in one group (the
             global-memory tie-group procedure), 1 025 - 4 096 in the next (the chunked staged scan and its bitonic
             order), tie groups longer than the ring's 2 048 events in flight (the stream restarts after the jump)
  long_runs  80 accelerators: every re-inserted leader leads a run of 79 tied events, processed 32 per step, longer than
             gsw_multi_kernel's 64-event walks and with more leaders than GSW_RUN_SLOTS
  open_walk  the same runs on rows that are all distinct: no tie group holds a second re-inserted leader, so every
             GE_MULTI flag comes from a walk that ran out of steps (the procedure is entered with one alive leader)
  long_jump  3 000 copies of which only the first three fail their first candidate: a 6 000-event tie group with three
             alive leaders at its start, jumped over in one step to the second class
  realistic  BASELINE configs[2]'s shape sized on the device with 30 % idle servers (GPU only)
  size limit S = 1 179 648 (the sweep's last covered size: GSW_ALIVE_WORDS x 32 alive bits) and S + 1 (the literal queue)

The CPU tests compute every fixture's static event list on the host (tau, sort, TIE / LEADER / CLS1 as
gsw_events_kernel / gsw_gather_kernel / gsw_multi_kernel form them), assert the shape each fixture promises, and check
the oracle's literal sorted-slice allocate() against the static-order formulation of policy None (restated here from
tools/proto/greedy_static_order.py; the proto itself is run where it is fast enough).  The GPU tests hold both
formulations under every policy to the oracle, bit for bit, and assert from the WVA_SIZER_DEBUG lines that the path each
fixture targets ran.
"""
import importlib.util
import os
import re
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = ("None", "PriorityExhaustive", "PriorityRoundRobin", "RoundRobin")
SOL_INT = ("state", "acc", "num_replicas", "batch_size")
F32_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_arrv_rate")
FLT_MAX = np.float32(np.finfo(np.float32).max)
SWEEP_MAX_SERVERS = 36 * 1024 * 32        # GSW_ALIVE_WORDS x 32 (greedy_sweep.cuh)
GSW_DYN_CAP, GSW_TIE_CAP, GSW_RUN_SLOTS, G_HEAP_SM = 4096, 1024, 8, 4096
RING_EVENTS = 4 * 512                      # GSW_SLOTS x GSW_BLOCK


# ---- fixtures ---------------------------------------------------------------------------------------------------
def _system(pkg, S, A, acc_type, prio, type_count):
    """A system whose candidates are installed from outside: one model per server, one instance and multiplicity 1 per
    replica (a candidate's demand is its replica count), capacity `type_count`."""
    d = pkg.synth.queue_system(S, A, 8, stream=900 + A)
    d["acc_type"] = np.asarray(acc_type, np.int32)
    d["n_types"] = len(type_count)
    d["type_count"] = np.asarray(type_count, np.int32)
    d["acc_multiplicity"] = np.ones(A, np.int32)
    d["perf_acc_count"] = np.ones((S, A), np.int32)
    d["srv_priority"] = np.asarray(prio, np.int32)
    d["unlimited"] = False
    return d


def _candidates(value, nrep, state=None):
    value = np.asarray(value, np.float32)
    S, A = value.shape
    rng = np.random.default_rng(S * 131 + A)
    c = {"state": np.ones((S, A), np.uint8) if state is None else np.asarray(state, np.uint8),
         "num_replicas": np.asarray(nrep, np.int32), "batch_size": rng.integers(1, 64, (S, A)).astype(np.int32),
         "cost": (value * np.float32(0.75) + np.float32(1.0)).astype(np.float32), "value": value,
         "n_solves": np.zeros((S, A), np.int32)}
    for k in ("itl", "ttft", "rho", "max_arrv_rate"):
        c[k] = rng.uniform(0.01, 100.0, (S, A)).astype(np.float32)
    return c


def _wide(pkg):
    """Class 1 (priority 1): 7 000 copies of the row (1, 9, 13, 15) — deltas 8 > 4 > 2, so ranks 1 and 2 lead re-inserted
    runs — with 1-4 replicas each (the order of the re-inserted leaders decides which servers get what).  Class 2
    (priority 5): 1 000 servers on 12 distinct rows."""
    rng = np.random.default_rng(11)
    n1, n2, A = 7000, 1000, 4
    S = n1 + n2
    value = np.empty((S, A), np.float32)
    value[:n1] = (1.0, 9.0, 13.0, 15.0)
    rows = np.array([np.sort(rng.choice(np.arange(1, 40), A, replace=False)) for _ in range(12)], np.float32)
    value[n1:] = rows[rng.integers(0, 12, n2)]
    nrep = rng.integers(1, 5, (S, A))
    prio = np.r_[np.full(n1, 1), np.full(n2, 5)]
    d1 = nrep[:n1].sum(0)
    # types 0-3 hold 12 %, 35 %, 30 %, 30 % of class 1's demand at ranks 0-3; the second class competes for what is left
    tc = [int(d1[0] * 0.12), int(d1[1] * 0.35), int(d1[2] * 0.3), int(d1[3] * 0.3)]
    return _system(pkg, S, A, np.arange(A), prio, tc), _candidates(value, nrep)


def _run_rows(offset, A):
    """(offset, offset + 1000, offset + 1001, ...): rank 1 leads a re-inserted run of A - 1 tied events."""
    v = np.empty((len(offset), A), np.float32)
    v[:, 0] = offset
    v[:, 1:] = np.asarray(offset, np.float32)[:, None] + 1000.0 + np.arange(A - 1, dtype=np.float32)[None, :]
    return v


def _run_nrep(rng, S, A):
    """Replicas falling along the run (90 at rank 1 down to 12), so a server fits deeper into its run the less is left."""
    nrep = np.empty((S, A), np.int64)
    nrep[:, 0] = rng.integers(2, 6, S)
    nrep[:, 1:] = np.maximum(90 - np.arange(A - 1)[None, :] + rng.integers(0, 3, (S, A - 1)), 12)
    return nrep


def _long_runs(pkg):
    """300 copies of one 80-candidate row: rank 0 on type 0 (fits 20 of them), ranks 1-79 one tied run on types 1-3."""
    rng = np.random.default_rng(12)
    S, A = 300, 80
    value = _run_rows(np.zeros(S, np.float32), A)
    nrep = _run_nrep(rng, S, A)
    acc_type = np.r_[0, 1 + np.arange(A - 1) % 3]
    tc = [int(np.sort(nrep[:, 0])[:20].sum()), 1500, 1500, 1500]
    return _system(pkg, S, A, acc_type, np.full(S, 1), tc), _candidates(value, nrep)


def _open_walk(pkg):
    """The long runs on 200 distinct rows: each tie group of a re-inserted run has exactly one leader."""
    rng = np.random.default_rng(13)
    S, A = 200, 80
    value = _run_rows(np.arange(S, dtype=np.float32) * 0.25, A)
    nrep = _run_nrep(rng, S, A)
    acc_type = np.r_[0, 1 + np.arange(A - 1) % 3]
    tc = [int(np.sort(nrep[:, 0])[:10].sum()), 1200, 1200, 1200]
    return _system(pkg, S, A, acc_type, np.full(S, 1), tc), _candidates(value, nrep)


def _long_jump(pkg):
    """Priority 1: 3 000 copies of (1, 9, 13); the first three servers want too much of type 0, everyone else fits there.
    Types 1 and 2 have room for one of the three each: the latest failure takes type 1, the next type 2, the first gets
    nothing.  Priority 5: 100 servers behind them on distinct rows (the stream goes on after the jump)."""
    rng = np.random.default_rng(14)
    n1, n2, A = 3000, 100, 3
    S = n1 + n2
    value = np.tile(np.array([1.0, 9.0, 13.0], np.float32), (S, 1))
    value[n1:] += np.arange(n2, dtype=np.float32)[:, None] * 0.5
    nrep = rng.integers(1, 4, (S, A))
    nrep[:3] = (10_000, 2, 1)
    tc = [int(nrep[3:n1, 0].sum()), 2, 1]
    prio = np.r_[np.full(n1, 1), np.full(n2, 5)]
    return _system(pkg, S, A, np.arange(A), prio, tc), _candidates(value, nrep)


def _size_limit(pkg, S):
    """A = 2, two types.  Priority 1 (all but the last 150 000 servers) fits on its first candidate; priority 5 (the last
    150 000, up to the last alive bit of the sweep) finds type 0 nearly exhausted, so about 100 000 of them fail it and
    are re-inserted at the front of the queue to test type 1 (popped at once: the oracle pays one vector::insert over
    the rest of the class each time)."""
    rng = np.random.default_rng(15)
    A, n2 = 2, 150_000
    n1 = S - n2
    base = rng.integers(0, 64, S).astype(np.float32)
    value = np.stack([base, base + rng.integers(1, 8, S).astype(np.float32)], 1)
    nrep = rng.integers(1, 4, (S, A))
    prio = np.r_[np.full(n1, 1), np.full(n2, 5)]
    tc = [int(nrep[:n1, 0].sum() + nrep[n1:, 0].sum() // 3), int(nrep[n1:, 1].sum() // 2)]
    return _system(pkg, S, A, np.arange(A), prio, tc), _candidates(value, nrep)


SYNTH = {"wide": _wide, "long_runs": _long_runs, "open_walk": _open_walk, "long_jump": _long_jump}
_CACHE = {}


def _fixture(pkg, name):
    if name not in _CACHE:
        _CACHE.clear()                                   # the size-limit systems are large: keep one fixture at a time
        if name.startswith("size_"):
            _CACHE[name] = _size_limit(pkg, int(name[5:]))
        else:
            _CACHE[name] = SYNTH[name](pkg)
    return _CACHE[name]


# ---- the static event list on the host ---------------------------------------------------------------------------
def _sortable(x):
    """float32 -> uint32, order-preserving, -0 == +0 (greedy_solve.cuh sortable_f32; the fixtures hold no NaN)"""
    x = np.asarray(x, np.float32).copy()
    x[x == 0] = 0.0
    b = x.view(np.uint32).astype(np.uint64)
    return np.where(b & 0x80000000, (~b) & 0xFFFFFFFF, b | 0x80000000).astype(np.uint64)


def events(sysd, cand):
    """Every potential event (server, rank) in the sweep's static order, with its flags.  Returns a dict of arrays."""
    S, A = int(sysd["n_servers"]), int(sysd["n_acc"])
    state = np.asarray(cand["state"]).reshape(S, A)
    value = np.asarray(cand["value"], np.float32).reshape(S, A)
    assert not np.isnan(value[state != 0]).any()
    order = np.argsort(np.where(state != 0, value, np.inf), axis=1, kind="stable")
    n = (state != 0).sum(1)
    j = np.arange(A)[None, :]
    ok = j < n[:, None]
    vs = np.take_along_axis(value, order, 1)
    nxt = np.concatenate([vs[:, 1:], np.zeros((S, 1), np.float32)], 1)
    delta = np.where(j + 1 < n[:, None], (nxt - vs).astype(np.float32), FLT_MAX)
    k = (((~_sortable(delta)) & 0xFFFFFFFF) << np.uint64(32)) | ((~_sortable(vs)) & 0xFFFFFFFF)
    k = np.where(ok, k, np.uint64(0))
    tau = np.maximum.accumulate(k, axis=1)
    prev = np.concatenate([np.zeros((S, 1), np.uint64), tau[:, :-1]], 1)
    leader = ok & ((j == 0) | (k > prev))
    cls1 = np.cumsum(leader & (j >= 1), axis=1) == 0
    model = np.asarray(sysd["srv_model"])
    acc = order
    live = (np.take_along_axis(state, order, 1) == 1) & (model[:, None] >= 0)
    inst = np.maximum(np.asarray(sysd["perf_acc_count"]).reshape(-1, A), 1)
    upr = np.take_along_axis(inst[np.maximum(model, 0)], order, 1).astype(np.int64) * np.asarray(sysd["acc_multiplicity"])[acc]
    typ = np.where(live, np.asarray(sysd["acc_type"])[acc], -1)
    cnt = np.where(live, np.take_along_axis(np.asarray(cand["num_replicas"]).reshape(S, A), order, 1).astype(np.int64) * upr, 0)
    srv = np.broadcast_to(np.arange(S)[:, None], (S, A))
    jj = np.broadcast_to(j, (S, A))
    prio = np.broadcast_to(np.asarray(sysd["srv_priority"]).astype(np.int64)[:, None], (S, A))
    last = jj == (n[:, None] - 1)
    f = {"srv": srv[ok], "j": jj[ok], "prio": prio[ok], "tau": tau[ok], "cls1": cls1[ok], "leader": leader[ok],
         "last": last[ok], "type": typ[ok], "cnt": cnt[ok], "acc": acc[ok]}
    # LSD as gsw_sweep's radix passes over (server, rank): run class, tau, priority
    o = np.lexsort((f["j"], f["srv"], f["cls1"], f["tau"], f["prio"]))
    f = {key: np.ascontiguousarray(v[o]) for key, v in f.items()}
    same = np.r_[False, (f["prio"][1:] == f["prio"][:-1]) & (f["tau"][1:] == f["tau"][:-1])]
    f["tie"] = same
    f["group"] = np.cumsum(~same) - 1
    return f


def multi_walks(f):
    """gsw_multi_kernel over the re-inserted leaders: (leaders whose walks found another leader, leaders whose walk ran
    64 events without finding one or the end of the part — the conservative GE_MULTI)."""
    tie, cls1, leader = f["tie"], f["cls1"], f["leader"]
    n = len(tie)
    found = opened = 0
    for i in np.flatnonzero(leader & ~cls1):
        multi = is_open = False
        k, steps = i + 1, 0
        while k < n and steps < 64:
            if not tie[k] or cls1[k]:
                break
            if leader[k]:
                multi = True
                break
            k += 1
            steps += 1
        if not multi and steps == 64:
            is_open = True
        if not multi:
            b, steps = i, 0
            while b > 0 and tie[b] and steps < 64:
                b -= 1
                steps += 1
                if cls1[b]:
                    break
                if leader[b]:
                    multi = True
                    break
            if not multi and steps == 64:
                is_open = True
        found += multi
        opened += is_open and not multi
    return found, opened


def static_sweep(sysd, f):
    """Policy None as the static-order sweep (tools/proto/greedy_static_order.py): groups of equal (priority, tau); a
    group whose re-inserted part holds two or more leaders takes its ALIVE leaders' runs latest insertion first, then its
    original entries.  Returns (accelerator per server or -1, statistics of the tie groups that needed the ordering)."""
    S = int(sysd["n_servers"])
    avail = [int(x) for x in sysd["type_count"]]
    srv, j, cls1, leader = f["srv"].tolist(), f["j"].tolist(), f["cls1"].tolist(), f["leader"].tolist()
    typ, cnt, acc, last, grp = f["type"].tolist(), f["cnt"].tolist(), f["acc"].tolist(), f["last"].tolist(), f["group"]
    alive = [True] * S
    stamp = [0] * S
    sel = np.full(S, -1, np.int64)
    clock = 0
    st = {"alive_leaders": [], "part_events": [], "jump": [], "max_run": 0, "n_groups": int(grp[-1]) + 1 if len(grp) else 0,
          "max_group": 0, "max_static_leaders": 0}

    def process(i):
        nonlocal clock
        e = srv[i]
        if not alive[e]:
            return False
        clock += 1
        t = typ[i]
        if t < 0:
            alive[e] = False
            return True
        if avail[t] >= cnt[i]:
            avail[t] -= cnt[i]
            sel[e] = acc[i]
            alive[e] = False
            return True
        stamp[e] = clock
        if last[i]:
            alive[e] = False
        return not alive[e]

    bounds = np.r_[np.flatnonzero(np.diff(grp)) + 1, len(grp)].tolist()
    g0 = 0
    for g1 in bounds:
        st["max_group"] = max(st["max_group"], g1 - g0)
        lead0 = [i for i in range(g0, g1) if leader[i] and not cls1[i]]
        st["max_static_leaders"] = max(st["max_static_leaders"], len(lead0))
        if len(lead0) >= 2:
            part_end = g0
            while part_end < g1 and not cls1[part_end]:
                part_end += 1
            act = [i for i in lead0 if alive[srv[i]]]
            if act:
                st["alive_leaders"].append(len(act))
                st["part_events"].append(part_end - g0)
                # events the sweep jumps from the first alive leader to the end of the part (0 when the part ends the list:
                # the sweep is over, nothing is streamed after it)
                st["jump"].append(part_end - act[0] if part_end < len(srv) else 0)
            act.sort(key=lambda i: -stamp[srv[i]])
            for i in act:
                e, k = srv[i], i
                while k < part_end and srv[k] == e:
                    done = process(k)
                    k += 1
                    if done:
                        break
                if len(act) >= 2:
                    st["max_run"] = max(st["max_run"], k - i)
            for i in range(part_end, g1):
                process(i)
        else:
            for i in range(g0, g1):
                process(i)
        g0 = g1
    return sel, st


def _proto():
    spec = importlib.util.spec_from_file_location("greedy_static_order", os.path.join(ROOT, "tools", "proto", "greedy_static_order.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _oracle_acc(o):
    return np.where(np.asarray(o["state"]) == 1, np.asarray(o["acc"]), -1)


# ---- CPU: shapes and the oracle against the static-order formulation -------------------------------------------------
def test_wide_shape_and_oracle(pkg, oracle):
    sysd, cand = _fixture(pkg, "wide")
    f = events(sysd, cand)
    sel, st = static_sweep(sysd, f)
    al = st["alive_leaders"]
    print("wide:", len(f["srv"]), "events,", st["n_groups"], "tie groups (largest", st["max_group"], "events), alive leaders",
          al, "parts", st["part_events"], "jumps", st["jump"])
    # one group past GSW_DYN_CAP and one between the staging size and GSW_DYN_CAP, both in priority class 1
    big = [k for k, a in enumerate(al) if a > GSW_DYN_CAP]
    mid = [k for k, a in enumerate(al) if GSW_TIE_CAP < a <= GSW_DYN_CAP]
    assert big and mid, al
    assert all(st["part_events"][k] > GSW_TIE_CAP for k in big + mid)
    assert max(st["jump"]) > RING_EVENTS
    assert len(np.unique(f["prio"])) == 2 and (f["prio"][f["leader"] & ~f["cls1"]] == 1).sum() > 2 * GSW_DYN_CAP
    lim = dict(sysd, saturation_policy="None")
    for delayed in (False, True):
        lim["delayed_best_effort"] = delayed
        assert np.array_equal(sel, _oracle_acc(oracle.solve(lim, cand))), delayed


def test_long_runs_shape_and_oracle(pkg, oracle):
    sysd, cand = _fixture(pkg, "long_runs")
    f = events(sysd, cand)
    sel, st = static_sweep(sysd, f)
    found, opened = multi_walks(f)
    print("long runs:", len(f["srv"]), "events, alive leaders", st["alive_leaders"], "longest run processed", st["max_run"],
          "walks: found a leader", found, "open", opened)
    assert int(sysd["n_acc"]) >= 65
    assert max(st["alive_leaders"]) > GSW_RUN_SLOTS
    assert st["max_run"] > 64                           # a run longer than two 32-event steps and than a 64-event walk
    assert opened > 0                                   # no second leader within 64 events: GE_MULTI by the open walk
    lim = dict(sysd, saturation_policy="None")
    for delayed in (False, True):
        lim["delayed_best_effort"] = delayed
        assert np.array_equal(sel, _oracle_acc(oracle.solve(lim, cand))), delayed


def test_open_walk_shape_and_oracle(pkg, oracle):
    sysd, cand = _fixture(pkg, "open_walk")
    f = events(sysd, cand)
    sel, st = static_sweep(sysd, f)
    found, opened = multi_walks(f)
    print("open walk:", len(f["srv"]), "events, largest tie group", st["max_group"], "walks: found a leader", found, "open", opened)
    assert st["max_static_leaders"] == 1 and found == 0 and opened > 0
    lim = dict(sysd, saturation_policy="None")
    ref, _, _ = _proto().static_greedy_none(lim, cand)
    assert np.array_equal(sel, ref)
    assert np.array_equal(sel, _oracle_acc(oracle.solve(lim, cand)))


def test_long_jump_shape_and_oracle(pkg, oracle):
    sysd, cand = _fixture(pkg, "long_jump")
    f = events(sysd, cand)
    sel, st = static_sweep(sysd, f)
    print("long jump: alive leaders", st["alive_leaders"], "parts", st["part_events"], "jumps", st["jump"])
    k = int(np.argmax(st["jump"]))
    assert st["jump"][k] > RING_EVENTS and 2 <= st["alive_leaders"][k] <= GSW_RUN_SLOTS
    lim = dict(sysd, saturation_policy="None")
    ref, _, _ = _proto().static_greedy_none(lim, cand)
    assert np.array_equal(sel, ref)
    assert np.array_equal(sel, _oracle_acc(oracle.solve(lim, cand)))


@pytest.mark.parametrize("S", [SWEEP_MAX_SERVERS, SWEEP_MAX_SERVERS + 1])
def test_size_limit_shape_and_oracle_time(pkg, oracle, S):
    sysd, cand = _fixture(pkg, f"size_{S}")
    f = events(sysd, cand)
    assert int(sysd["n_servers"]) == S and len(f["srv"]) == 2 * S
    lim = dict(sysd, saturation_policy="None", delayed_best_effort=False)
    t0 = time.perf_counter()
    o = oracle.solve(lim, cand)
    dt = time.perf_counter() - t0
    un = np.asarray(o["state"]) == 0
    n2 = 150_000
    refit = ((np.asarray(o["acc"]) == 1) & ~un)[-n2:].sum() + un[-n2:].sum()    # failed rank 0: re-inserted once each
    print(f"size limit S={S}: oracle {dt:.1f} s, {int(refit)} re-insertions, {int(un.sum())} unallocated")
    assert 50_000 < refit < 150_000 and un[-n2:].any()


# ---- GPU: both formulations, every policy, against the oracle ---------------------------------------------------
_SWEEP_RE = re.compile(r"tie-group calls (\d+).*tie groups: (\d+) over the staging size \((\d+) events\), (\d+) in global memory, "
                       r"alive leaders (\d+) \(max (\d+)\).*stream restarts (\d+)")


def _stats(err):
    """Counters of the greedy debug lines of one solve: the sweep's (None when it did not run) and the queue's heap."""
    m = _SWEEP_RE.search(err)
    sweep = None
    if m:
        sweep = dict(zip(("tie_calls", "staged_over", "staged_over_events", "global", "alive", "max_alive", "restarts"),
                         map(int, m.groups())))
    h = re.search(r"greedy queue: .*largest heap (\d+)", err)
    return sweep, (int(h.group(1)) if h else None)


def _check(g, o, tag):
    for k in SOL_INT:
        assert np.array_equal(g[k], o[k]), (k, tag, np.argwhere(np.asarray(g[k]) != np.asarray(o[k]))[:5])
    for k in F32_FIELDS:
        assert np.array_equal(np.ascontiguousarray(g[k]).view(np.uint8), np.ascontiguousarray(o[k]).view(np.uint8)), (k, tag)
    assert np.array_equal(g["type_count"], o["type_count"]), tag


def _all_policies(engine, oracle, capfd, sysd, cand, tag):
    """Every policy x delayed under both formulations (WVA_OPT_GREEDY_MODE 2 sweep, 1 literal queue), each against the
    oracle.  Returns the debug counters of every run: {(mode, policy, delayed): (sweep, largest heap)}."""
    engine.load_system(sysd)
    engine.set_candidates(cand)
    out = {}
    try:
        for policy in POLICIES:
            for delayed in (False, True):
                o = oracle.solve(dict(sysd, saturation_policy=policy, delayed_best_effort=delayed), cand)
                assert (np.asarray(o["state"]) == 0).any()                 # the cap binds
                for mode in (2, 1):
                    engine.set_option(5, mode)
                    engine.set_optimizer(False, delayed, policy)
                    capfd.readouterr()
                    engine.solve()
                    err = capfd.readouterr().err
                    _check(engine.solution(), o, (tag, mode, policy, delayed))
                    out[(mode, policy, delayed)] = _stats(err)
    finally:
        engine.set_option(5, 0)
    return out


def _sweeps(runs):
    s = [v[0] for (mode, _, _), v in runs.items() if mode == 2]
    assert all(x is not None for x in s)
    return s


@pytest.mark.gpu
def test_wide_tie_groups_gpu(pkg, engine, oracle, capfd, monkeypatch):
    """More than 4 096 alive leaders (global-memory procedure), a staged group past the staging size, stream restarts;
    the literal queue's heap past its shared-memory slots.  Prints the solve time of both formulations."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    sysd, cand = _fixture(pkg, "wide")
    runs = _all_policies(engine, oracle, capfd, sysd, cand, "wide")
    for s in _sweeps(runs):
        assert s["global"] >= 1 and s["max_alive"] > GSW_DYN_CAP, s
        assert s["staged_over"] >= 1 and s["restarts"] >= 1, s
    heaps = [v[1] for (mode, _, _), v in runs.items() if mode == 1]
    assert all(h is not None and h > G_HEAP_SM for h in heaps), heaps
    # device time of the solve (sweep and queue, policy None), CUDA events around wva_solve
    monkeypatch.delenv("WVA_SIZER_DEBUG")
    engine.set_optimizer(False, False, "None")
    times = {}
    try:
        for mode in (2, 1):
            engine.set_option(5, mode)
            engine.solve()
            ms = []
            for _ in range(5):
                engine.solve()
                ms.append(engine.timing()["solve_ms"])
            times[mode] = float(np.median(ms))
    finally:
        engine.set_option(5, 0)
    import torch
    print(f"\nwide tie groups ({torch.cuda.get_device_name(0)}): solve {times[2]:.2f} ms with the event sweep, "
          f"{times[1]:.2f} ms with the literal queue (median of 5)")


@pytest.mark.gpu
def test_long_runs_gpu(pkg, engine, oracle, capfd, monkeypatch):
    """Re-inserted runs of 79 tied events, more alive leaders than run slots: the staged procedure's run steps."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    sysd, cand = _fixture(pkg, "long_runs")
    runs = _all_policies(engine, oracle, capfd, sysd, cand, "long_runs")
    for s in _sweeps(runs):
        assert s["tie_calls"] >= 1 and GSW_RUN_SLOTS < s["max_alive"] <= GSW_DYN_CAP and s["global"] == 0, s


@pytest.mark.gpu
def test_open_walk_gpu(pkg, engine, oracle, capfd, monkeypatch):
    """No tie group holds two re-inserted leaders: the procedure runs only because a 64-event walk stayed open, and
    then finds one alive leader."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    sysd, cand = _fixture(pkg, "open_walk")
    runs = _all_policies(engine, oracle, capfd, sysd, cand, "open_walk")
    for s in _sweeps(runs):
        assert s["tie_calls"] >= 1 and s["max_alive"] == 1, s


@pytest.mark.gpu
def test_long_jump_gpu(pkg, engine, oracle, capfd, monkeypatch):
    """Three alive leaders at the start of a 6 000-event tie group: the sweep jumps past the events in flight."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    sysd, cand = _fixture(pkg, "long_jump")
    runs = _all_policies(engine, oracle, capfd, sysd, cand, "long_jump")
    for s in _sweeps(runs):
        assert s["restarts"] >= 1 and s["staged_over"] >= 1 and 2 <= s["max_alive"] <= GSW_RUN_SLOTS, s


@pytest.mark.gpu
def test_realistic_idle_fleet_gpu(pkg, engine, oracle, capfd, monkeypatch):
    """BASELINE configs[2]'s shape (100 000 servers x 32) with 30 % idle servers, sized on the device and capped at half
    the demand: identical idle candidates form tie groups past the staging size (about 170 tie-group calls, 3 of them
    scanned in chunks, at most 11 alive leaders: the global-memory procedure needs the synthesized fixtures).  The
    oracle's greedy takes the device's candidates."""
    d = pkg.synth.queue_system(100_000, 32, 8, stream=177, zero_load_frac=0.3)
    engine.load_system(d)
    engine.calculate()
    cand = engine.candidates()
    engine.set_optimizer(True)
    engine.solve()
    lim = pkg.synth.limit_capacity(d, engine.solution()["type_count"], 0.5)
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    runs = _all_policies(engine, oracle, capfd, lim, cand, "realistic")
    s = _sweeps(runs)
    print("\nrealistic:", s[0])
    assert all(x["tie_calls"] >= 1 and x["staged_over"] >= 1 for x in s), s


@pytest.mark.gpu
@pytest.mark.parametrize("S", [SWEEP_MAX_SERVERS, SWEEP_MAX_SERVERS + 1])
def test_size_limit_switches_formulation_gpu(pkg, engine, oracle, capfd, monkeypatch, S):
    """At 1 179 648 servers the default is the event sweep, one more server and it is the literal queue; the default
    equals the forced other formulation (where there is one) and the oracle."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    sysd, cand = _fixture(pkg, f"size_{S}")
    engine.load_system(sysd)
    engine.set_candidates(cand)
    try:
        for policy, delayed in (("None", False), ("PriorityExhaustive", True), ("RoundRobin", False)):
            o = oracle.solve(dict(sysd, saturation_policy=policy, delayed_best_effort=delayed), cand)
            engine.set_optimizer(False, delayed, policy)
            for mode in (0, 1, 2):
                engine.set_option(5, mode)
                capfd.readouterr()
                engine.solve()
                err = capfd.readouterr().err
                _check(engine.solution(), o, (S, mode, policy, delayed))
                sweep_ran = "greedy sweep:" in err
                # mode 1 forces the queue; 0 (default) and 2 take the sweep wherever it covers the system
                assert sweep_ran == (mode != 1 and S <= SWEEP_MAX_SERVERS), (S, mode, err[-300:])
                assert ("greedy queue:" in err) == (not sweep_ran)
    finally:
        engine.set_option(5, 0)
