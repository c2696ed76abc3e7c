"""The head of the greedy sweep: the events before the first failure, committed in parallel.

Up to the first failure P of the static-order sweep (greedy_sweep.cuh) every alive event is an entry's first candidate:
it is taken, or dropped when it has no accelerator.  P is the first rank-0 event on a type t >= 0 at which the running
sum of the rank-0 units of type t passes the capacity.  The sweep's nothing-fits check can stop it earlier, at a block
start C < P; the device commits the events before C = min(P, that block start) at once and sweeps on from C.

Fixtures: systems whose first S events are all rank-0 candidates (every rank-0 delta is larger than every later one),
with the capacity placed so that P lands where a case wants it: the first event, the middle of a 512-event block, a
block start, a priority boundary, inside a tie group, after entries with no accelerator, nowhere (nothing fails), and
nowhere with the capacity used up by the first candidates, where the nothing-fits check stops the sweep first.  Then fleet-shaped systems of
10 000 and 100 000 servers over up to 64 types, sized on the device.

The CPU tests restate P and C with numpy over the static event list, check them against a sequential walk of the list
and check that the oracle gives every first candidate before P to its server.  The GPU tests hold the sweep (and the
literal queue) to the oracle bit for bit under every policy, and the device's P and C (WVA_SIZER_DEBUG line) to the
host's.
"""
import re

import numpy as np
import pytest

from tests.test_fleet_systems import _limited, fleet_system
from tests.test_greedy_ties import POLICIES, _candidates, _check, _system, events

GSW_BLOCK = 512


# ---- fixtures ---------------------------------------------------------------------------------------------------------
def _rows(rng, S, A):
    """Sorted candidate values with a rank-0 gap (>= 100) larger than every later gap (<= 8): every first candidate sorts
    before every other event of its priority class.  Accelerators are permuted per server, so first candidates spread
    over the types."""
    v0 = rng.integers(0, 50, S).astype(np.float32)
    v = np.empty((S, A), np.float32)
    v[:, 0] = v0
    v[:, 1] = v0 + 100.0 + rng.integers(0, 20, S)
    for j in range(2, A):
        v[:, j] = v[:, j - 1] + rng.integers(1, 9, S)
    perm = np.argsort(rng.random((S, A)), axis=1)
    out = np.empty_like(v)
    np.put_along_axis(out, perm, v, axis=1)
    return out


def _base(pkg, seed, S=3000, A=3, prio=None, unknown=(), dup=0):
    """S servers on A accelerators (type = accelerator); `dup` servers copy server 0's row (one tie group of first
    candidates); `unknown` servers run an unknown model (no accelerator behind any candidate)."""
    rng = np.random.default_rng(seed)
    value = _rows(rng, S, A)
    value[1:1 + dup] = value[0]
    nrep = rng.integers(1, 6, (S, A))
    prio = np.full(S, 1) if prio is None else prio
    sysd = _system(pkg, S, A, np.arange(A), prio, [1] * A)
    sysd["srv_model"] = sysd["srv_model"].copy()
    sysd["srv_model"][list(unknown)] = -1
    return sysd, _candidates(value, nrep)


def _place_p(sysd, f, i, slack=0):
    """Capacities under which the first failure is event i.  The other types keep what the rank-0 events up to i want
    plus a third of the rest, so the capacity still binds after P.  i = len(events): every type holds what its rank-0
    events want, plus `slack`."""
    T = int(sysd["n_types"])
    first = (f["j"] == 0) & (f["type"] >= 0)
    cap = np.zeros(T, np.int64)
    for t in range(T):
        m = first & (f["type"] == t)
        upto = f["cnt"][: i + 1][m[: i + 1]].sum()
        rest = f["cnt"][i + 1:][m[i + 1:]].sum()
        cap[t] = upto + rest // 3
    if i < len(f["srv"]):
        t = f["type"][i]
        assert first[i] and f["cnt"][i] >= 1
        cap[t] = f["cnt"][: i + 1][first[: i + 1] & (f["type"][: i + 1] == t)].sum() - 1
    else:
        cap = np.array([f["cnt"][first & (f["type"] == t)].sum() + slack for t in range(T)], np.int64)
    sysd = dict(sysd)
    sysd["type_count"] = cap.astype(np.int32)
    return sysd


def head(sysd, f):
    """(P, C) restated over the static event list: P the first rank-0 event whose type's running rank-0 sum passes the
    capacity, C = min(P, the first block start at which no event of any type from there on fits the capacity left)."""
    n, T = len(f["srv"]), int(sysd["n_types"])
    cap = np.asarray(sysd["type_count"], np.int64)
    typ, cnt = f["type"], f["cnt"].astype(np.int64)
    first = (f["j"] == 0) & (typ >= 0)
    P = n
    for t in range(T):
        idx = np.flatnonzero(first & (typ == t))
        over = idx[np.cumsum(cnt[idx]) > cap[t]]
        if len(over):
            P = min(P, int(over[0]))
    nb = n // GSW_BLOCK + 1
    blk = np.arange(n) // GSW_BLOCK
    big = np.iinfo(np.int64).max
    bmin = np.full((nb, T), big, np.int64)
    has = typ >= 0
    np.minimum.at(bmin, (blk[has], typ[has]), cnt[has])
    suf = np.minimum.accumulate(bmin[::-1], axis=0)[::-1]
    bsum = np.zeros((nb, T), np.int64)
    np.add.at(bsum, (blk[first], typ[first]), cnt[first])
    left = cap[None, :] - (np.cumsum(bsum, axis=0) - bsum)     # capacity left at each block start, nothing failed before
    fits = ((suf != big) & (left >= 0) & (left >= suf)).any(axis=1)
    stops = np.flatnonzero(~fits)
    C = min(P, int(stops[0]) * GSW_BLOCK) if len(stops) else P
    return P, min(C, n)


def walk_to_first_failure(sysd, f):
    """The sequential sweep (alive bits and capacities, event by event) up to its first failure: (position, the
    accelerator each server got before it)."""
    S = int(sysd["n_servers"])
    avail = np.asarray(sysd["type_count"], np.int64).copy()
    alive = np.ones(S, bool)
    got = np.full(S, -1, np.int64)
    for i in range(len(f["srv"])):
        e = f["srv"][i]
        if not alive[e]:
            continue
        t = f["type"][i]
        if t >= 0 and avail[t] < f["cnt"][i]:
            return i, got
        assert f["j"][i] == 0
        alive[e] = False
        if t >= 0:
            avail[t] -= f["cnt"][i]
            got[e] = f["acc"][i]
    return len(f["srv"]), got


def _case(pkg, name):
    """(system, candidates, static events) of one case; the capacity places P."""
    if name == "nothing_fits_first":
        # every type holds exactly what its first candidates want: nothing fails, and at the first block start after
        # the first candidates nothing is left for any later one: the nothing-fits check stops the sweep before P
        sysd, cand = _base(pkg, 41)
        f = events(sysd, cand)
        return _place_p(sysd, f, len(f["srv"])), cand, f
    if name == "priority_boundary":
        S, n1 = 3000, 900
        sysd, cand = _base(pkg, 42, prio=np.r_[np.full(n1, 1), np.full(S - n1, 5)])
        f = events(sysd, cand)
        i = n1 * 3                                       # class 1's events (3 per server), then class 2's first one
        assert f["prio"][i] == 5 and f["prio"][i - 1] == 1
        return _place_p(sysd, f, i), cand, f
    if name == "tie_group":
        sysd, cand = _base(pkg, 43, dup=200)
        f = events(sysd, cand)
        i = int(np.flatnonzero(f["tie"] & (f["j"] == 0) & (f["srv"] <= 200))[100])   # in the middle of the 201 copies
        return _place_p(sysd, f, i), cand, f
    if name == "unknown_before":
        sysd, cand = _base(pkg, 44, unknown=range(0, 3000, 7))
        f = events(sysd, cand)
        i = int(np.flatnonzero((f["j"] == 0) & (f["type"] >= 0) & (np.arange(len(f["srv"])) >= 1500))[0])
        assert ((f["type"][:i] < 0) & (f["j"][:i] == 0)).sum() > 100
        return _place_p(sysd, f, i), cand, f
    sysd, cand = _base(pkg, 45)
    f = events(sysd, cand)
    n = len(f["srv"])
    i = {"first_event": 0, "mid_block": GSW_BLOCK + 300, "block_start": 2 * GSW_BLOCK, "none_fails": n}[name]
    return _place_p(sysd, f, i, slack=100_000), cand, f


CASES = ["first_event", "mid_block", "block_start", "priority_boundary", "tie_group", "unknown_before", "none_fails",
         "nothing_fits_first"]


# ---- CPU ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_head_restatement(pkg, oracle, name):
    """numpy's P and C against the sequential walk and the case's promise; the oracle gives every first candidate
    before P to its server."""
    sysd, cand, f = _case(pkg, name)
    n = len(f["srv"])
    P, C = head(sysd, f)
    walked, got = walk_to_first_failure(sysd, f)
    assert P == walked
    want = {"first_event": 0, "mid_block": GSW_BLOCK + 300, "block_start": 2 * GSW_BLOCK, "none_fails": n}
    if name in want:
        assert P == want[name] and C == P
    elif name == "nothing_fits_first":
        assert P == n and C == 3072 and (f["j"][:3000] == 0).all()
    else:
        assert C == P and 0 < P < n
        if name == "priority_boundary":
            assert f["prio"][P] != f["prio"][P - 1]
        if name == "tie_group":
            assert f["tie"][P] and f["srv"][P] in range(201)
        if name == "unknown_before":
            assert P % GSW_BLOCK != 0
    o = oracle.solve(dict(sysd, saturation_policy="None", delayed_best_effort=False), cand)
    acc = np.where(np.asarray(o["state"]) == 1, np.asarray(o["acc"]), -1)
    done = got >= 0
    assert np.array_equal(acc[done], got[done])


# ---- GPU ---------------------------------------------------------------------------------------------------------------
_HEAD_RE = re.compile(r"head: first failure at (-?\d+), (\d+) first candidates committed in parallel, swept from (\d+) to (\d+)")


def _device_head(err):
    m = _HEAD_RE.findall(err)
    assert len(m) == 1, err[-2000:]
    return tuple(int(x) for x in m[0])


def _solve_all(engine, oracle, capfd, sysd, cand, policies, tag, installed=True):
    """every policy x delayed, sweep (mode 2) and literal queue (mode 1), against the oracle; returns the device's head
    counters of every sweep"""
    heads = []
    try:
        for policy in policies:
            for delayed in (False, True):
                o = oracle.solve(dict(sysd, saturation_policy=policy, delayed_best_effort=delayed), cand)
                for mode in (2, 1):
                    engine.set_option(5, mode)
                    engine.set_capacity(sysd["type_count"])
                    engine.set_optimizer(False, delayed, policy)
                    capfd.readouterr()
                    engine.solve()
                    err = capfd.readouterr().err
                    _check(engine.solution(), o, (tag, mode, policy, delayed))
                    if mode == 2:
                        heads.append(_device_head(err))
    finally:
        engine.set_option(5, 0)
    return heads


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_head_matches_oracle_gpu(pkg, engine, oracle, capfd, monkeypatch, name):
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    sysd, cand, f = _case(pkg, name)
    P, C = head(sysd, f)
    engine.load_system(sysd)
    engine.set_candidates(cand)
    heads = _solve_all(engine, oracle, capfd, sysd, cand, POLICIES, name)
    first = int(((f["j"][:C] == 0)).sum())
    for dp, committed, start, stop in heads:
        assert (dp, start, committed) == (P, C, first), (name, dp, start, committed, P, C, first)
        assert start <= stop


def _fleet(pkg, engine, S, M, A, T, seed, n_max):
    d = fleet_system(S, M, A, T, seed=seed, n_max=n_max)
    engine.load_system(d)
    engine.calculate()
    cand = engine.candidates()
    engine.set_optimizer(True)
    engine.solve()
    un = engine.solution()
    return _limited(pkg, d, un["type_count"], 0.6), cand


@pytest.mark.gpu
@pytest.mark.parametrize("S,M,A,T,policies", [(10_000, 120, 40, 64, POLICIES),
                                                (100_000, 400, 32, 64, ("None", "PriorityRoundRobin"))])
def test_fleet_head_matches_oracle_gpu(pkg, engine, oracle, capfd, monkeypatch, S, M, A, T, policies):
    """fleet-shaped systems sized on the device, capacity 60 % of the unlimited demand: the solution against the oracle,
    the device's P and C against the host's restatement over the same candidates"""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    lim, cand = _fleet(pkg, engine, S, M, A, T, seed=700 + T, n_max=64)
    f = events(lim, cand)
    P, C = head(lim, f)
    heads = _solve_all(engine, oracle, capfd, lim, cand, policies, f"fleet {S}")
    assert P < len(f["srv"])                             # the capacity binds (at 10 k servers over 64 types, at once)
    for dp, committed, start, stop in heads:
        assert (dp, start) == (P, C), (dp, start, P, C)
        assert committed == int((f["j"][:C] == 0).sum())
