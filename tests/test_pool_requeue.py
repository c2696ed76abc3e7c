"""The pool sizer queues the solves its fast solve (E12) does not certify for exact batches of their own instead of
redoing them in the batch that tried them.  Forced pool sizer (set_option(1, 6)) on systems that put those exact
batches through their corner cases: every candidate bit-equal to the oracle, and the counts equal to the host replay."""
import numpy as np
import pytest

from tests.test_fast_solve import F32_FIELDS, GRID_CASES, _bit_equal, _boundary_grid_system, fast  # noqa: F401


def _pool_calculate(engine, sysd):
    engine.set_option(1, 6)
    try:
        engine.load_system(sysd)
        engine.calculate()
        return engine.candidates(), engine.timing()
    finally:
        engine.set_option(1, 0)


def _check_oracle(g, o):
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(g[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k


def _check_counts(t, replay):
    solves, fallbacks, ovf, window = replay
    print("%d solves, %d not certified (device %d), %d pairs to the slow path" %
          (solves, fallbacks, t["certify_fallbacks"], t["overflow_pairs"]))
    assert t["chain_solves"] == solves
    assert t["certify_fallbacks"] == fallbacks
    assert t["overflow_pairs"] == ovf + window


@pytest.mark.gpu
@pytest.mark.parametrize("N,R,S,A,stream", GRID_CASES)
def test_requeue_on_boundary_systems(pkg, engine, oracle, fast, N, R, S, A, stream):
    """Arrival rates placed next to float32 rounding boundaries of the fast solve's statistics."""
    sysd = _boundary_grid_system(pkg, fast, N, R, S, A, stream)
    g, t = _pool_calculate(engine, sysd)
    _check_oracle(g, oracle.calculate(sysd))
    _check_counts(t, fast.calculate(sysd)["_counts"])


@pytest.mark.gpu
@pytest.mark.parametrize("N,S,A,stream", [(1, 400, 8, 31), (1200, 24, 6, 32)])
def test_requeue_with_many_fallbacks(pkg, engine, oracle, fast, N, S, A, stream):
    """N = 1 has no head, so every solve is queued for an exact batch (thousands of full exact batches); N = 1200 grows
    past the exponent window on some solves, which the exact batch hands to the slow path."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    g, t = _pool_calculate(engine, sysd)
    _check_oracle(g, oracle.calculate(sysd))
    replay = fast.calculate(sysd)["_counts"]
    _check_counts(t, replay)
    if N == 1:
        assert replay[1] == replay[0] > 32 * 64


@pytest.mark.gpu
@pytest.mark.parametrize("S,A", [(1, 1), (3, 2)])
def test_requeue_drains_partial_exact_batches(pkg, engine, oracle, fast, S, A):
    """A system too small to fill an exact class (N = 1: every solve is queued, fewer than 32 at a time): the partial
    exact batches are taken once no fast request is left, and the kernel ends."""
    sysd = pkg.synth.queue_system(S, A, 1, stream=41, zero_load_frac=0.0, infeasible_frac=0.0)
    g, t = _pool_calculate(engine, sysd)
    _check_oracle(g, oracle.calculate(sysd))
    _check_counts(t, fast.calculate(sysd)["_counts"])
    assert t["certify_fallbacks"] == t["chain_solves"] > 0


def _mixed_system(pkg, S, A, stream, nil_frac=0.0, zero_frac=0.05):
    sysd = pkg.synth.queue_system(S, A, 256, stream=stream, zero_load_frac=zero_frac)
    rng = np.random.default_rng(stream)
    sysd["srv_max_batch"] = rng.choice(np.array([1, 2, 31, 33, 256, 1200], np.int32), S)
    if nil_frac:
        sysd["perf_present"] = (rng.random((S, A)) >= nil_frac).astype(np.uint8)
    return sysd


@pytest.mark.gpu
def test_requeue_mixed_batch_sizes(pkg, engine, oracle):
    """N in {1, 2, 31, 33, 256, 1200} in one pool: fast and exact classes hold requests of several N, and batches of
    mixed N take the per-lane state machine."""
    sysd = _mixed_system(pkg, 240, 8, 51)
    g, t = _pool_calculate(engine, sysd)
    _check_oracle(g, oracle.calculate(sysd))


@pytest.mark.gpu
def test_requeue_with_nil_and_zero_load_pairs(pkg, engine, oracle):
    """Pairs without a performance profile (nil) and servers without load are settled in setup, lane by lane, between
    pairs whose rows the warp builds together."""
    sysd = _mixed_system(pkg, 240, 8, 52, nil_frac=0.3, zero_frac=0.3)
    g, t = _pool_calculate(engine, sysd)
    _check_oracle(g, oracle.calculate(sysd))
