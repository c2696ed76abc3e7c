"""Replica grid at its edges, against the oracle bit for bit: the launch shapes by batch size, replica counts around the
warp width and the 16-bit deferral limit, a deferral list far past its capacity, chains that overflow float64, stale
device buffers between runs; and, on the CPU, the oracle's own float64 rescale path against a log-domain reference."""
import math
import re

import numpy as np
import pytest

from tests.test_gpu_parity import _bit_equal

F32 = np.float32
DBL_MAX_LOG = math.log(np.finfo(np.float64).max)
LN2 = math.log(2.0)


def _compare(g, o, full=True):
    assert np.array_equal(g["frontier"], o["frontier"]), np.argwhere(g["frontier"] != o["frontier"])[:5]
    if full:
        assert np.array_equal(g["ok"], o["ok"]), np.argwhere(g["ok"] != o["ok"])[:5]
        for k in ("ttft", "itl", "rho", "tput"):
            assert _bit_equal(g[k], o[k]), (k, np.argwhere(g[k].view(np.uint32) != o[k].view(np.uint32))[:5])


def _grid_matches(engine, oracle, sysd, R, o=None):
    """full grid and frontier-only grid of one system, both against the oracle; returns the oracle's grid"""
    engine.load_system(sysd)
    o = oracle.analyze_grid(sysd, R) if o is None else o
    _compare(engine.analyze_grid(R), o)
    engine.grid_run(R, full=False)
    assert np.array_equal(engine.grid_fetch_frontier(), o["frontier"])
    return o


def _with_defer(engine, mode, fn):
    engine.set_option(6, mode)
    try:
        return fn()
    finally:
        engine.set_option(6, 0)


# ---- float32 restatement of the grid's per-pair setup (grid_setup, model_init, serv_rate, analyze_admits) --------------
def _f(x):
    return F32(x)


def _pair_model(sysd, srv, acc):
    """(N, K, float32 head table mu_1..mu_N, rate_max) as BuildModel forms them, or None for a pair without levels"""
    arrival = sysd["srv_arrival"][srv]
    in_tok, out_tok = int(sysd["srv_in_tokens"][srv]), int(sysd["srv_out_tokens"][srv])
    m = sysd["srv_model"][srv]
    if arrival <= 0 or out_tok == 0 or not sysd["perf_present"][m, acc] or not sysd["srv_target_present"][srv]:
        return None
    N = int(sysd["srv_max_batch"][srv]) or max(1, int(sysd["perf_max_batch"][m, acc]) * int(sysd["perf_at_tokens"][m, acc]) // out_tok)
    a, b, g = (_f(sysd[k][m, acc]) for k in ("perf_alpha", "perf_beta", "perf_gamma"))
    I, O = _f(in_tok), _f(out_tok)
    tc = _f(_f(I + O) / _f(O + _f(1)))
    tm = _f(I + _f(O / _f(2)))
    slope = _f(_f(b * tc) + _f(g * tm))
    pre_c = _f(_f(b + g) * I)
    dec_c = _f(g * tm)
    n = np.arange(1, N + 1, dtype=F32)
    it = (a + n * slope).astype(F32)
    pre = np.zeros(N, F32) if in_tok == 0 else (it + pre_c).astype(F32)
    dec = (O * ((it + b).astype(F32) + dec_c).astype(F32)).astype(F32)
    mu = (n / (pre + dec).astype(F32)).astype(F32)
    lmax = _f(mu[-1] * _f(_f(1) - _f(0.001)))
    return N, N + 10 * N, mu, _f(lmax * _f(1000))


def _log_terms(mu, K, lam):
    """log p~[0..K] of the chain p~[n+1] = p~[n] lam / mu[min(n, N-1)], p~[0] = 1, in float64"""
    idx = np.minimum(np.arange(K), len(mu) - 1)
    return np.concatenate(([0.0], np.cumsum(math.log(float(lam)) - np.log(mu[idx].astype(np.float64)))))


def _classify_levels(sysd, R, thr=0.6):
    """For every admitted level of the system: whether the grid defers it (ratio lambda / mu_N > thr, deferral forced) and
    how its chain behaves in float64 — 'term' (a term overflows), 'sum' (only the sum does), 'window' (leaves the E3
    window [2^-500, 2^500) without overflowing) or 'plain'.  Levels within a margin of a boundary are 'edge'."""
    out = []
    S, A = len(sysd["srv_arrival"]), int(sysd["n_acc"])
    for srv in range(S):
        for acc in range(A):
            pm = _pair_model(sysd, srv, acc)
            if pm is None:
                continue
            N, K, mu, rate_max = pm
            total = _f(_f(sysd["srv_arrival"][srv]) / _f(60))
            for r in range(1, R + 1):
                rate = _f(total / _f(r))
                if not (rate > 0 and not rate > rate_max):
                    continue
                lam = _f(rate / _f(1000))
                deferred = bool(_f(lam / mu[-1]) > _f(thr))
                lt = _log_terms(mu, K, lam)
                top = lt.max() / LN2                                    # log2 of the largest term
                tot = np.logaddexp.reduce(lt) / LN2                     # log2 of the sum
                x = top + math.log2(float(lam))                         # log2 of the largest p~ * lambda
                if top > 1025:
                    kind = "term"
                elif top < 1023 and tot > 1025:
                    kind = "sum"
                elif 505 < x and top < 1023 and tot < 1023:
                    kind = "window"
                elif x < 480 and tot < 480:
                    kind = "plain"
                else:
                    kind = "edge"
                out.append((srv, acc, r, deferred, kind))
    return out


def _alpha_system(pkg, rows, A=2, alphas=(4.0, 3.0)):
    """Alpha-dominated servers (beta = gamma = 0, no input tokens, 16 output tokens: mu_n = n / (16 alpha)), the shape
    whose chains overflow float64 from N ~ 710 on; rows = [(N, total rate in req/s)]"""
    S = len(rows)
    sysd = pkg.synth.queue_system(S, A, 16, stream=31, zero_load_frac=0.0, infeasible_frac=0.0)
    sysd["perf_alpha"][:] = np.array(alphas[:A], F32)[None, :]
    sysd["perf_beta"][:] = 0.0
    sysd["perf_gamma"][:] = 0.0
    sysd["srv_in_tokens"][:] = 0
    sysd["srv_out_tokens"][:] = 16
    sysd["perf_at_tokens"][:] = 16
    sysd["srv_max_batch"][:] = [n for n, _ in rows]
    sysd["srv_arrival"][:] = [60.0 * t for _, t in rows]
    sysd["srv_slo_ttft"][:] = 5000.0
    sysd["srv_slo_itl"][:] = 0.0
    sysd["srv_slo_tps"][:] = 0.0
    return sysd


# N = 1024 at 160 000 req/s (R = 64): r <= 10 not admitted, 11-14 a term overflows, 15-29 leave the exponent window,
# from 30 on plain; deferred (lambda / mu_N > 0.6) up to r = 16.  N = 1500 and 2047 put overflowing levels below the
# deferral ratio too (a term overflows from lambda / mu_N ~ 0.35 on at N = 2047); at 100 000 req/s and r = 9 the N = 2047
# chain's largest term is 2^1019.9 and its sum 2^1025.9.  N = 64 adds plain deferred levels.
OVERFLOW_ROWS = [(1024, 160000.0), (1500, 70000.0), (2047, 100000.0), (64, 16000.0)]
OVERFLOW_R = 64


def test_overflow_system_reaches_every_chain_kind(pkg):
    """CPU: the overflow system below has, in the main and in the deferred pass, levels whose terms overflow, levels that
    leave the exponent window and plain levels, and at least one level where only the sum crosses DBL_MAX."""
    lv = _classify_levels(_alpha_system(pkg, OVERFLOW_ROWS), OVERFLOW_R)
    for deferred in (False, True):
        kinds = {k for *_, d, k in lv if d == deferred}
        assert {"term", "window", "plain"} <= kinds, (deferred, kinds)
    assert any(k == "sum" for *_, k in lv)
    assert any(k == "sum" and not d for *_, d, k in lv)


# ---- launch shapes -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_grid_mixed_batch_sizes_in_the_one_warp_launch(pkg, engine, oracle):
    """N = 2548 selects grid_kernel<1>; the same system's N = 1, 2 and 33 pairs run inside it, and the deferred pass
    (forced) sees items of four batch sizes."""
    sysd = pkg.synth.queue_system(16, 3, 33, stream=41, R=96)
    sysd["srv_max_batch"][:] = np.array([1, 2, 33, 2548], np.int32)[np.arange(16) % 4]
    o = oracle.analyze_grid(sysd, 96)
    assert o["ok"].any()
    for mode in (2, 1):
        _with_defer(engine, mode, lambda: _grid_matches(engine, oracle, sysd, 96, o))


@pytest.mark.gpu
def test_grid_batch_size_above_the_limit_is_refused(pkg, engine, oracle):
    """N = 10189 needs more shared memory per warp than an SM has: WVA_ERR_LIMIT, and the engine still computes the
    next system's grid correctly."""
    sysd = pkg.synth.queue_system(3, 2, 10189, stream=42, R=8)
    engine.load_system(sysd)
    with pytest.raises(pkg.WvaError, match="10188"):
        engine.analyze_grid(8)
    nxt = pkg.synth.queue_system(3, 2, 10188, stream=43, R=8)
    _grid_matches(engine, oracle, nxt, 8)


# ---- replica counts around the 16-bit deferral item ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("R", [65535, 65536])
def test_grid_replica_counts_at_the_deferral_item_limit(pkg, engine, oracle, R):
    """Deferred items pack r into 16 bits: R = 65535 still defers (forced), R = 65536 turns deferral off and runs
    every level in the main pass.  Small N keeps the oracle cheap; arrival rates put admitted and deferred levels
    near r = R."""
    sysd = pkg.synth.queue_system(4, 2, 2, stream=44, R=R, zero_load_frac=0.0, infeasible_frac=0.0)
    sysd["srv_max_batch"][:] = [1, 2, 1, 2]
    # total rate = f R mu_N: levels r >= f R / 0.999 are admitted, those below f R / 0.6 deferred
    mu_n = np.array([[_pair_model(sysd, s, a)[2][-1] for a in range(2)] for s in range(4)], np.float64).max(axis=1)
    sysd["srv_arrival"][:] = 60.0 * 1000.0 * R * mu_n * np.array([0.95, 0.5, 0.3, 0.62])
    o = oracle.analyze_grid(sysd, R)
    assert o["ok"][:, :, -1].any() and not o["ok"].all()
    _with_defer(engine, 2, lambda: _grid_matches(engine, oracle, sysd, R, o))


# ---- deferral list past its capacity --------------------------------------------------------------------------------
def _heavy_system(pkg, S, A, N, R, stream):
    """Every accelerator of a server runs the same perf, and each server's load puts lambda / mu_N above the deferral
    ratio on ~0.4 R of its levels: far more deferred levels than the list's 16 per pair."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream, R=R, zero_load_frac=0.0, infeasible_frac=0.0)
    for k in ("perf_alpha", "perf_beta", "perf_gamma"):
        sysd[k][:] = sysd[k][:, :1]
    mu_n = np.array([_pair_model(sysd, s, 0)[2][-1] for s in range(S)], np.float64)
    t = np.random.default_rng(stream).uniform(0.4, 0.6, S) * R            # total rate / mu_N, in levels
    sysd["srv_arrival"][:] = 60.0 * 1000.0 * t * mu_n
    return sysd


def _reserved(err):
    m = re.findall(r"deferral reserved (\d+) of capacity (\d+)", err)
    assert m, err
    return [(int(a), int(b)) for a, b in m]


@pytest.mark.gpu
def test_grid_deferral_list_past_capacity(pkg, oracle, capfd, monkeypatch):
    """Forced deferral on a system that asks for several times the list's 16 P + 1024 slots: the warp whose reservation
    crosses the capacity defers only the lanes that fit and solves the rest, later warps solve everything in place.
    Fresh engine first; then the same system right after a larger one, whose items and rows still fill the reused
    device buffers."""
    monkeypatch.setenv("WVA_SIZER_DEBUG", "1")
    small = _heavy_system(pkg, 40, 8, 32, 512, stream=45)
    large = _heavy_system(pkg, 64, 8, 32, 1024, stream=46)
    o_small = oracle.analyze_grid(small, 512)
    o_large = oracle.analyze_grid(large, 1024)
    eng = pkg.Engine(device=0)
    try:
        eng.set_option(6, 2)
        capfd.readouterr()
        _grid_matches(eng, oracle, small, 512, o_small)
        res = _reserved(capfd.readouterr().err)
        _grid_matches(eng, oracle, large, 1024, o_large)
        res += _reserved(capfd.readouterr().err)
        _grid_matches(eng, oracle, small, 512, o_small)
        res += _reserved(capfd.readouterr().err)
    finally:
        eng.close()
    print("deferral reservations / capacity:", [f"{a}/{b} = {a / b:.1f}x" for a, b in res])
    # full and frontier-only run of each system; capacity min(P R, 16 P + 1024)
    assert [b for _, b in res] == [16 * 320 + 1024] * 2 + [16 * 512 + 1024] * 2 + [16 * 320 + 1024] * 2
    for a, b in res:
        assert a >= 2 * b, (a, b)


# ---- stale buffers ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_grid_runs_reuse_buffers(pkg, engine, oracle):
    """Large-R full grid, then a smaller frontier-only grid, then the full grid again on the same engine: each run
    writes every output and frontier it reports, whatever the last one left in the reused buffers."""
    big = pkg.synth.queue_system(24, 6, 64, stream=47, R=300)
    small = pkg.synth.queue_system(10, 3, 16, stream=48, R=20)
    ob = oracle.analyze_grid(big, 300)
    os_ = oracle.analyze_grid(small, 20, full=False)
    for mode in (2, 1):
        def run():
            engine.load_system(big)
            _compare(engine.analyze_grid(300), ob)
            engine.load_system(small)
            engine.grid_run(20, full=False)
            assert np.array_equal(engine.grid_fetch_frontier(), os_["frontier"])
            _compare(engine.analyze_grid(20, full=False), os_, full=False)
            engine.load_system(big)
            engine.grid_run(300, full=False)
            assert np.array_equal(engine.grid_fetch_frontier(), ob["frontier"])
        _with_defer(engine, mode, run)


# ---- chains that overflow float64 ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_grid_float64_overflow_levels_match_oracle(pkg, engine, oracle, mode):
    """Levels whose chain overflows float64 get the reference's metrics (computeProbabilities rescales), not ok = 0:
    the overflow pass solves them with literal_solve.  Mode 2 defers the near-saturation levels, so both the main and
    the deferred kernel meet overflowing, window-leaving and plain levels (test_overflow_system_reaches_every_chain_kind)."""
    sysd = _alpha_system(pkg, OVERFLOW_ROWS)
    o = oracle.analyze_grid(sysd, OVERFLOW_R)
    _with_defer(engine, mode, lambda: _grid_matches(engine, oracle, sysd, OVERFLOW_R, o))
    n_ovf = sum(k in ("term", "sum") for *_, k in _classify_levels(sysd, OVERFLOW_R))
    assert engine.timing()["overflow_pairs"] == n_ovf > 0


@pytest.mark.gpu
def test_grid_overflow_list_capacity_is_an_error(pkg, engine, oracle):
    """One pair with more overflowing levels than the overflow list's 16 P + 1024: the run fails with WVA_ERR_LIMIT
    instead of dropping levels, and the engine then computes the next grid correctly."""
    R = 6000
    sysd = _alpha_system(pkg, [(1024, 160000.0 * 400)], A=1)
    engine.load_system(sysd)
    with pytest.raises(pkg.WvaError, match="overflow list"):
        engine.grid_run(R, full=False)
    _grid_matches(engine, oracle, _alpha_system(pkg, OVERFLOW_ROWS), OVERFLOW_R)


# ---- CPU: the oracle's float64 rescale path against a log-domain reference -----------------------------------------
U = 2.0 ** -53


def _overflow_cases():
    N = 1024
    mu = (np.arange(1, N + 1, dtype=F32) / F32(64)).astype(F32)         # alpha = 4, 16 output tokens: mu_n = n / 64
    cases = [(f"r{r}", _f(_f(_f(F32(160000)) / _f(r)) / _f(1000))) for r in (11, 12, 13, 14, 15, 20, 29)]
    cases.append(("sum", _f(_f(_f(F32(100000.0)) / _f(9)) / _f(1000))))  # peak term below DBL_MAX, sum above
    return N, mu, cases


@pytest.mark.parametrize("case", [c for c, _ in _overflow_cases()[2]])
def test_oracle_rescale_path_matches_log_domain(oracle, case):
    """oracle_statedep_solve on N = 1024 chains whose terms (r11-r14) or only whose sum ('sum') overflow float64, and on
    chains that only leave the exponent window (r15-r29), against exp(log p~[n] - logsumexp(log p~)) in float64."""
    N, mu, cases = _overflow_cases()
    lam = dict(cases)[case]
    if case == "sum":
        mu = (np.arange(1, 2048, dtype=F32) / F32(64)).astype(F32)      # the N = 2047 server of OVERFLOW_ROWS at r = 9
        N = len(mu)
    K = N + 10 * N
    rc, rows, p = oracle.statedep_solve(K, mu, [lam])
    assert rc == 0, "pathological: the reference would never leave its rescale loop"
    st = rows[0]
    assert st["valid"] == 1.0

    terms = math.log(float(lam)) - np.log(mu[np.minimum(np.arange(K), N - 1)].astype(np.float64))
    L = np.concatenate(([0.0], np.cumsum(terms)))
    top = L.max()
    lse = top + math.log(np.exp(L - top).sum())
    if case.startswith("r1") and int(case[1:]) <= 14:
        assert top > DBL_MAX_LOG                          # a term overflows: the p[n+1] rescale branch
    elif case == "sum":
        assert top < DBL_MAX_LOG - 1 and lse > DBL_MAX_LOG + 1   # only the running sum crosses DBL_MAX
    ref = np.exp(L - lse)

    # Tolerance, relative, per state n.  The reference: each log term errs by <= 2u(|log lam| + |log mu|), each cumsum
    # step by u |L[k]|, so L[n] by e[n] = sum_{k<=n} (u |L[k]| + 2u(|log lam| + |log mu_k|)).  logsumexp moves by the
    # softmax-weighted sum of those, sum_n p[n] e[n], plus its own roundings: exp(L - top) by u(1 + |L - top|) each, the
    # K-term sum by K u, the final log and addition by 2u |lse|.  The subtraction and exp add u |L[n] - lse| + u.  The
    # cumulative sum dominates: ~1e-9 at the far end of the states above 2^-900.  The oracle: n multiplications and n
    # divisions per p~[n] (2n u), a few divisions by the rescale factor, a K-term sum and the normalisation ((K + 70) u).
    e_term = 2 * U * (abs(math.log(float(lam))) + np.abs(np.log(mu[np.minimum(np.arange(K), N - 1)].astype(np.float64))))
    eL = np.concatenate(([0.0], np.cumsum(U * np.abs(L[1:]) + e_term)))
    w = np.exp(L - lse)
    e_lse = float((w * (eL + U * (1 + np.abs(L - top)))).sum()) + K * U + 2 * U * abs(lse)
    n = np.arange(K + 1)
    tol = 1.01 * (eL + e_lse + U * np.abs(L - lse) + U + (2 * n + K + 70) * U)
    keep = ref > 2.0 ** -900
    rel = np.abs(p[keep] / ref[keep] - 1.0)
    print(f"{case}: {keep.sum()} states above 2^-900, largest relative error {rel.max():.2e}, "
          f"largest tolerance {tol[keep].max():.2e}")
    assert tol[keep].max() < 2e-9
    assert (rel <= tol[keep]).all(), (np.argmax(rel - tol[keep]), rel.max())
    # p[n] below 2^-900 carry the normalisation's underflow; they must still be tiny
    assert np.all(p[~keep] <= 2.0 ** -899)

    # statistics (computeStatistics), float64 from the reference p; 1 - sumP_N as the tail sum (no cancellation)
    Lsys = float((n * ref).sum())
    Lserv = float((n[: N + 1] * ref[: N + 1]).sum() + N * ref[N + 1:].sum())
    X = float(lam) * (1.0 - float(ref[K]))
    for k, v in (("throughput", X), ("avgNumInServers", Lserv), ("avgNumInSystem", Lsys)):
        assert abs(st[k] - v) <= 1e-6 * abs(v), (k, st[k], v)
    # avgWaitTime = f32(L32 / X32) - f32(Ls32 / X32): each float32 value and quotient errs by 2^-24 relative, so the two
    # quotients by <= 3 * 2^-24 of L / X and Ls / X each and their difference by another 2^-24 of W; that is the
    # cancellation's bound, plus 1e-8 relative for the float64 reference under it.
    W = max(0.0, (Lsys - Lserv) / X)
    tolW = 2.0 ** -24 * (3 * (Lsys + Lserv) / X + W) + 1e-8 * (Lsys + Lserv) / X
    assert abs(st["avgWaitTime"] - W) <= tolW, (st["avgWaitTime"], W, tolW)
