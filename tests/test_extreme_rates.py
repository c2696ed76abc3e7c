"""Sizing and the replica grid at service rates outside the (E1) divisor range [2^-126, 2^126], against the oracle bit
for bit.

The coefficients are accepted at load time (finite and >= 0) and the reference answers them, but the device's reciprocal
seed rcp.approx.ftz.f32 flushes there: mu in (2^126, 2^128) has a subnormal 1/mu (seed 0), a subnormal mu reads as 0, and
mu = +inf (all-zero perf coefficients) gives a NaN reciprocal.  Pairs with such a rate divide with the IEEE division on
every state (PairModel::e1_ok); these tests hold every sizer, table mode and grid pass to the oracle on them, next to
ordinary pairs in the same warps and pools."""
import numpy as np
import pytest

from tests.test_grid_edges import _grid_matches, _pair_model, _with_defer

F32_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_arrv_rate")
F32 = np.float32


def _extreme(sysd, rows, alpha, gamma, arrival, out_tok=16, N=32):
    """servers `rows` of sysd: beta = 0, no input tokens, out_tok output tokens, max batch N, the given alpha / gamma
    (per accelerator or scalar) and arrival rate (req/min).  With alpha = 0 and 16 output tokens,
    mu_n = n / (128 gamma (n + 1)); with gamma = 0 and one output token, mu_n = n / alpha."""
    sysd["perf_alpha"][rows] = alpha
    sysd["perf_beta"][rows] = 0.0
    sysd["perf_gamma"][rows] = gamma
    sysd["srv_in_tokens"][rows] = 0
    sysd["srv_out_tokens"][rows] = out_tok
    sysd["perf_at_tokens"][rows] = out_tok
    sysd["perf_max_batch"][rows] = N
    sysd["srv_max_batch"][rows] = N
    sysd["srv_arrival"][rows] = arrival
    sysd["perf_present"][rows] = 1
    sysd["srv_target_present"][rows] = 1
    if np.all(np.asarray(alpha) == 0) and np.all(np.asarray(gamma) == 0):
        # mu = +inf: RateRange.Max is inf, and every solve of the sizer's searches runs at lambda = inf, a NaN chain that
        # spins in the reference's rescale loop up to its guard on every state; without SLO targets there are two
        # solves per pair instead of ~30
        sysd["srv_slo_ttft"][rows] = 0.0
        sysd["srv_slo_itl"][rows] = 0.0


# (alpha, gamma, arrival, output tokens, N) and the service rates mu_1 .. mu_N each recipe gives
RECIPES = {
    "high": (0.0, 3.4438e-41, 1e38, 16, 32),        # all in (2^126.4, 2^127.5)
    "straddle": (0.0, 5.5102e-41, 1e38, 16, 32),    # mu_1 below 2^126, the rest above
    "inf": (0.0, 0.0, 600.0, 16, 32),               # +inf
    "subnormal": (3e38, 0.0, 2e-34, 1, 3),          # float32 subnormals 3.3e-39, 6.7e-39, 1e-38
    "subnormal_head": (3e38, 0.0, 1e-33, 1, 32),    # mu_1 .. mu_3 subnormal, the rest normal
    "control": (0.0, 2.0 ** -110, 1e30, 16, 32),    # 2^102 .. 2^103
}


def _recipe_system(pkg, name, S=4, A=3, stream=61):
    sysd = pkg.synth.queue_system(S, A, 32, stream=stream, zero_load_frac=0.0, infeasible_frac=0.0)
    _extreme(sysd, slice(None), *RECIPES[name])
    return sysd


def _mixed_system(pkg, S=48, A=4, stream=62):
    """queue_system pairs with every fourth server made extreme, a different recipe per server, so that extreme and
    ordinary pairs share warps, lane tables and pool batches (all pairs have N = 32)"""
    sysd = pkg.synth.queue_system(S, A, 32, stream=stream, zero_load_frac=0.0, infeasible_frac=0.0)
    sysd["srv_max_batch"][:] = 32
    names = list(RECIPES)
    for k, srv in enumerate(range(1, S, 4)):
        _extreme(sysd, [srv], *RECIPES[names[k % len(names)]])
    # one extreme server whose accelerators differ: high, +inf, subnormal head, ordinary
    srv = S - 2
    _extreme(sysd, [srv], 0.0, 0.0, 1e-33, 1, 32)
    sysd["perf_alpha"][srv] = [0.0, 0.0, 3e38, 4.0]
    sysd["perf_beta"][srv] = [0.0, 0.0, 0.0, 0.1]
    sysd["perf_gamma"][srv] = [2.2e-39, 0.0, 0.0, 0.01]
    return sysd


def _same(a, b):
    """float32 arrays equal bit for bit, except that any NaN equals any NaN: a pair sized at lambda = inf (RateRange.Max
    overflows float32) reports NaN in max_arrv_rate, and the device's NaN (0x7fffffff) is not the x86 host's (0xffc00000)"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    both_nan = np.isnan(a) & np.isnan(b)
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | both_nan))


def _rate_max_finite(sysd):
    """every sized pair's RateRange.Max is finite in float32: no solve runs at lambda = inf, where the reference's chain
    is NaN and takes its rescale branch"""
    S, A = len(sysd["srv_arrival"]), int(sysd["n_acc"])
    for s in range(S):
        for a in range(A):
            pm = _pair_model(sysd, s, a)
            if pm is not None and not np.isfinite(pm[3]):
                return False
    return True


def _service_rates(sysd, srv, acc):
    return _pair_model(sysd, srv, acc)[2]


def test_recipes_reach_their_service_rates(pkg):
    """CPU: each recipe puts the service rates where its name says, on every pair."""
    for name in RECIPES:
        sysd = _recipe_system(pkg, name)
        mu = _service_rates(sysd, 0, 0).astype(np.float64)
        if name == "high":
            assert (mu > 2.0 ** 126).all() and (mu < 2.0 ** 128).all()
        elif name == "straddle":
            assert mu[0] < 2.0 ** 126 < mu[1]
        elif name == "inf":
            assert np.isinf(mu).all()
        elif name == "subnormal":
            assert (mu > 0).all() and (mu < 2.0 ** -126).all()
        elif name == "subnormal_head":
            assert (mu[:3] > 0).all() and (mu[:3] < 2.0 ** -126).all() and (mu[3:] > 2.0 ** -126).all()
        else:
            assert (mu >= 2.0 ** 102).all() and (mu < 2.0 ** 104).all()


def _systems(pkg):
    out = [(name, _recipe_system(pkg, name)) for name in RECIPES]
    out.append(("mixed", _mixed_system(pkg)))
    return out


_ORACLE = {}


def _oracle_calc(oracle, name, sysd):
    if name not in _ORACLE:
        _ORACLE[name] = oracle.calculate(sysd)
    return _ORACLE[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RECIPES) + ["mixed"])
def test_calculate_at_extreme_rates_matches_oracle(pkg, engine, oracle, name):
    """calculate under every sizer (WVA_OPT_FORCE_LANE_SIZER 0-6: 0 picks the warp sizer at this size, 6 is the pool)
    and both lane-table modes (WVA_OPT_TABLE_MODE 1, 2): state, replicas, batch size and every float32 field equal the
    oracle's bit for bit (NaN payloads aside).  Where no solve runs at lambda = inf, no pair goes to the float64 overflow path."""
    sysd = dict(_systems(pkg))[name]
    o = _oracle_calc(oracle, name, sysd)
    no_rescale = _rate_max_finite(sysd)
    try:
        for table in (1, 2):
            engine.set_option(4, table)
            for sizer in range(7):
                engine.set_option(1, sizer)
                engine.load_system(sysd)
                engine.calculate()
                g = engine.candidates()
                t = engine.timing()
                where = (name, sizer, table)
                for k in ("state", "num_replicas", "batch_size"):
                    assert np.array_equal(g[k], o[k]), (where, k, np.argwhere(g[k] != o[k])[:5])
                for k in F32_FIELDS:
                    assert _same(g[k], o[k]), (where, k, np.argwhere(g[k].view(np.uint32) != o[k].view(np.uint32))[:5])
                if no_rescale:
                    assert t["overflow_pairs"] == 0, (where, t["overflow_pairs"])
    finally:
        engine.set_option(1, 0)
        engine.set_option(4, 0)
    print(f"{name}: {int((o['state'] == 1).sum())} feasible candidates; rescale-free sizing: {no_rescale}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RECIPES) + ["mixed"])
@pytest.mark.parametrize("R", [16, 40, 64])
def test_grid_at_extreme_rates_matches_oracle(pkg, engine, oracle, name, R):
    """analyze_grid with deferral off (mode 1) and forced (mode 2), full and frontier-only: ok, ttft, itl, rho, tput and
    the frontier equal the oracle's, and no level goes to the overflow pass (every level's lambda is finite, and none
    of these chains overflows float64)."""
    sysd = dict(_systems(pkg))[name]
    o = oracle.analyze_grid(sysd, R)
    assert o["ok"].any()
    for mode in (1, 2):
        _with_defer(engine, mode, lambda: _grid_matches(engine, oracle, sysd, R, o))
        assert engine.timing()["overflow_pairs"] == 0, (name, R, mode)
    if name == "high" and R == 64:
        print("high: rho[0, 0, :3] =", o["rho"][0, 0, :3])


@pytest.mark.gpu
def test_zero_coefficient_grid_past_the_overflow_list(pkg, engine, oracle):
    """2,000 pairs with all-zero perf coefficients (mu = +inf) at R = 64: 128,000 levels, more than the overflow list's
    16 P + 1024 = 33,024.  Every level is solved in place (p~[1] = lambda / inf = 0) and the grid equals the oracle's
    (ok, rho = itl = 0, frontier 1) instead of failing with WVA_ERR_LIMIT."""
    R = 64
    sysd = pkg.synth.queue_system(1000, 2, 32, stream=63, zero_load_frac=0.0, infeasible_frac=0.0)
    _extreme(sysd, slice(None), 0.0, 0.0, 600.0)
    sysd["srv_slo_tps"][:] = 0.0
    o = oracle.analyze_grid(sysd, R)
    assert o["ok"].all() and (o["frontier"] == 1).all()
    for mode in (0, 2):
        _with_defer(engine, mode, lambda: _grid_matches(engine, oracle, sysd, R, o))
        assert engine.timing()["overflow_pairs"] == 0
