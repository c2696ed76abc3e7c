"""The pool sizer and the deferred grid pass keep no head table: each solve computes its pair's service rates from the
model's coefficients (RateTable in lockstep_solve.cuh; model_rate for the per-lane chain of mixed-N batches, of pairs
outside the (E1) divisor range and of the slow paths).  Forced pool sizer (set_option(1, 6)) and forced deferral
(set_option(6, 2)) on the systems whose rates take each of those paths: every candidate and grid field equal to the
oracle bit for bit, and where the host replay models the pool's batches (one N, inside the exponent window) its solve
and fallback counts too."""
import numpy as np
import pytest

from tests.test_extreme_rates import _mixed_system as _extreme_mixed_system, _same
from tests.test_fast_solve import F32_FIELDS, fast  # noqa: F401
from tests.test_grid_edges import _grid_matches, _pair_model, _with_defer
from tests.test_pool_requeue import _check_counts, _pool_calculate


def _check_oracle(g, o):
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(g[k], o[k]), (k, np.argwhere(g[k] != o[k])[:5])
    for k in F32_FIELDS:
        assert _same(g[k], o[k]), (k, np.argwhere(g[k].view(np.uint32) != o[k].view(np.uint32))[:5])


def _small_n_system(pkg, S=160, A=6, stream=71):
    """N in {1, 2, 17, 33}: one fast class (N <= 38), so its batches mix batch sizes and take the per-lane chain"""
    sysd = pkg.synth.queue_system(S, A, 33, stream=stream)
    sysd["srv_max_batch"] = np.random.default_rng(stream).choice(np.array([1, 2, 17, 33], np.int32), S)
    return sysd


def _non_monotone_system(pkg, S=6, A=2, stream=72):
    """N = 4096 with a service rate that dips under float32 rounding near the top of the head: mono > 0 on every pair
    (n / (7e-3 (n 7/8 + 1)) changes by less than an ulp per state there)"""
    sysd = pkg.synth.queue_system(S, A, 4096, stream=stream, zero_load_frac=0.0, infeasible_frac=0.0)
    sysd["perf_alpha"][:] = 0.0
    sysd["perf_beta"][:] = 1e-3
    sysd["perf_gamma"][:] = 0.0
    sysd["srv_in_tokens"][:] = 0
    sysd["srv_out_tokens"][:] = 7
    sysd["perf_at_tokens"][:] = 7
    sysd["srv_max_batch"][:] = 4096
    return sysd


def _no_input_system(pkg, S=120, A=6, stream=73):
    """half the servers without input tokens: PrefillTime is 0 (queueanalyzer.go:268-273) in their rates"""
    sysd = pkg.synth.queue_system(S, A, 256, stream=stream)
    sysd["srv_in_tokens"][::2] = 0
    return sysd


def _mono(mu):
    """the last descent !(mu[n-1] <= mu[n]), as BuildModel's scan finds it"""
    d = np.nonzero(~(mu[:-1] <= mu[1:]))[0]
    return int(d[-1]) + 1 if d.size else 0


def test_non_monotone_system_has_descents(pkg):
    """CPU: the non-monotone recipe really dips (mono > 0) and keeps every rate an (E1) divisor."""
    sysd = _non_monotone_system(pkg)
    for srv in range(len(sysd["srv_arrival"])):
        mu = _pair_model(sysd, srv, 0)[2].astype(np.float64)
        assert 0 < _mono(mu) < len(mu)
        assert ((mu >= 2.0 ** -126) & (mu <= 2.0 ** 126)).all()


SYSTEMS = {"small_n": _small_n_system, "non_monotone": _non_monotone_system, "no_input": _no_input_system}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SYSTEMS))
def test_pool_sizer_computed_rates(pkg, engine, oracle, fast, name):
    """The replay's counts hold for "no_input" only: a mixed-N batch solves on the per-lane chain without a fast solve
    (the replay counts every N = 1 solve as not certified), and the N = 4096 pairs leave the float64 exponent window,
    where the pool retires a pair at its first such solve."""
    sysd = SYSTEMS[name](pkg)
    g, t = _pool_calculate(engine, sysd)
    _check_oracle(g, oracle.calculate(sysd))
    if name == "no_input":
        _check_counts(t, fast.calculate(sysd)["_counts"])


@pytest.mark.gpu
def test_pool_sizer_rates_outside_e1(pkg, engine, oracle):
    """Pairs with a service rate outside [2^-126, 2^126] next to ordinary ones in the same pool: the warp's scan flags
    them (e1_ok = 0) and their solves run on the per-lane chain, every candidate as the oracle's."""
    sysd = _extreme_mixed_system(pkg)
    g, _ = _pool_calculate(engine, sysd)
    _check_oracle(g, oracle.calculate(sysd))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SYSTEMS) + ["outside_e1"])
def test_deferred_grid_computed_rates(pkg, engine, oracle, name):
    """Every deferred level solved from the pair's coefficients, full grid and frontier-only, with deferral forced."""
    R = 64
    sysd = _extreme_mixed_system(pkg) if name == "outside_e1" else SYSTEMS[name](pkg)
    o = oracle.analyze_grid(sysd, R)
    _with_defer(engine, 2, lambda: _grid_matches(engine, oracle, sysd, R, o))
