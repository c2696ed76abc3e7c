"""The certified fast chain solve (DESIGN.md §3, E12) on the host build of the device core: one head pass plus a
closed-form tail, accepted only where an error enclosure proves the reference's float32 statistics."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_arrv_rate")


@pytest.fixture(scope="module")
def fast(pkg, tmp_path_factory):
    """tests/host_emul/fast_emul.cpp (emul.cpp plus the fast-solve replays), built into a temporary directory."""
    src = os.path.join(ROOT, "tests", "host_emul", "fast_emul.cpp")
    so = str(tmp_path_factory.mktemp("fast_emul") / "libfastemul.so")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-pthread",
                    "-shared", "-o", so, src], check=True)
    lib = C.CDLL(so)
    abi = pkg._abi
    lib.emul_check_fast_solve.argtypes = [C.c_int64, C.c_uint64, C.c_int, C.POINTER(C.c_int64)]
    lib.emul_fast_boundary.argtypes = [C.c_int64, C.c_uint64, C.c_int, C.c_double, C.POINTER(C.c_int64)]
    lib.emul_calculate_fast.argtypes = [C.POINTER(abi.System), C.POINTER(abi.Candidates), C.POINTER(C.c_int64)]
    lib.emul_grid_deferred.argtypes = [C.POINTER(abi.System), C.c_int, C.c_float] + [C.c_void_p] * 6 + [C.POINTER(C.c_int64)]
    lib.emul_grid_boundary_arrival.argtypes = [C.POINTER(abi.System), C.c_int, C.c_int, C.c_float, C.c_float, C.c_int]
    lib.emul_grid_boundary_arrival.restype = C.c_float

    def check(n, seed, N):
        st = (C.c_int64 * 5)()
        lib.emul_check_fast_solve(n, seed, N, st)
        return list(st)

    def boundary(n, seed, N, band):
        st = (C.c_int64 * 5)()
        lib.emul_fast_boundary(n, seed, N, band, st)
        return list(st)

    def calculate(sysd):
        st, keep = abi.make_system(sysd)
        cst, cand = abi.alloc_candidates(st.n_servers, st.n_acc)
        counts = (C.c_int64 * 4)()
        lib.emul_calculate_fast(C.byref(st), C.byref(cst), counts)
        cand["_counts"] = list(counts)
        return cand

    def grid(sysd, R, thr):
        st, keep = abi.make_system(sysd)
        n = st.n_servers * st.n_acc
        out = {"ok": np.zeros(n * R, np.uint8), "frontier": np.zeros(n, np.int32)}
        for k in ("ttft", "itl", "rho", "tput"):
            out[k] = np.zeros(n * R, np.float32)
        counts = (C.c_int64 * 4)()
        lib.emul_grid_deferred(C.byref(st), R, thr, *[out[k].ctypes.data for k in ("ok", "ttft", "itl", "rho", "tput",
                                                                                    "frontier")], counts)
        for k in list(out):
            out[k] = out[k].reshape(st.n_servers, st.n_acc, *(() if k == "frontier" else (R,)))
        out["_counts"] = list(counts)
        return out

    def boundary_arrival(sysd, srv, R, thr, ratio0, max_steps):
        st, keep = abi.make_system(sysd)
        return float(lib.emul_grid_boundary_arrival(C.byref(st), srv, R, thr, ratio0, max_steps))

    lib.check, lib.boundary, lib.calculate, lib.grid, lib.boundary_arrival = check, boundary, calculate, grid, boundary_arrival
    return lib


def _bit_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def test_fast_solve_matches_literal_chain(fast):
    """10^6 random solves of configs[2]-shaped models, half of them at lambda / lambda_max in [0.95, 1]: no certified
    lane differs in any bit from the literal chain solver, and at most 10^-3 of the lanes with N >= 2 fall back, not
    counting the solves whose head terms leave the float64 exponent window (at N = 1200 the head grows past 2^500 for
    ~12 % of the draws: the exact lock-step solver hands those to the literal slow path too).  N = 1 has no head and
    is always left to the exact solver."""
    total = {"cert": 0, "fallback": 0}
    for N, n, seed in ((1, 20_000, 1), (7, 450_000, 2), (32, 450_000, 3), (256, 100_000, 4), (1200, 10_000, 5)):
        cert, fallback, diff, ovf, window = fast.check(n, seed, N)
        assert diff == 0, (N, cert, diff)
        assert cert + fallback + ovf == n
        if N == 1:
            assert cert == 0
            continue
        fallback -= window
        assert fallback <= 1e-3 * (cert + fallback), (N, cert, fallback, window)
        total["cert"] += cert
        total["fallback"] += fallback
    assert total["cert"] + total["fallback"] >= 1_000_000
    print("fast solve: %d certified, %d fallbacks (rate %.2e)" %
          (total["cert"], total["fallback"], total["fallback"] / (total["cert"] + total["fallback"])))


def test_fast_solve_refuses_rounding_boundaries(fast):
    """Solves whose reference L or Lserv sits next to a float32 rounding boundary (found with the literal solver):
    within the a-priori floor of the enclosure none is certified, and within 10^-11 none is certified wrongly."""
    near, cert, wrong, floor_hits, floor_cert = fast.boundary(2_000_000, 17, 7, 1e-11)
    assert near > 50 and wrong == 0, (near, cert, wrong)
    assert floor_hits > 0 and floor_cert == 0, (floor_hits, floor_cert)


@pytest.mark.parametrize("S,A,N,stream", [(10, 4, 32, 1), (40, 8, 16, 7), (12, 6, 128, 2), (4, 4, 256, 3),
                                          (20, 3, 1, 11), (16, 3, 5, 12)])
def test_fast_solve_state_machine_matches_oracle(pkg, oracle, fast, S, A, N, stream):
    """The whole sizer state machine with the fast solve reproduces CreateAllocation bit for bit."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    e = fast.calculate(sysd)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k
    solves, fallbacks, ovf, _ = e["_counts"]
    assert ovf == 0 and solves > 0
    if N >= 2:
        assert fallbacks <= 0.05 * solves, (solves, fallbacks)


# ---- the device certifies what the host replay certifies --------------------------------------------------------
# The pool sizer (sizer_pool_kernel) and the deferred grid pass (grid_deferred_kernel) run lockstep_solve_fast, which
# forms q0 differently from the host replay fast_solve (p (lambda r) against (p lambda) r: E1 makes p~ the same bits)
# and keeps lanes that left the head early running with lambda = 0.  Outputs equal to the oracle do not show that both
# certify the same solves: the exact fallback gives the same bits.  The fallback counters do.

# (N, S, A, stream): one batch size per system, so every pool batch is uniform and takes the fast solve
POOL_CASES = [(1, 40, 6, 11), (2, 40, 6, 12), (17, 40, 6, 13), (18, 40, 6, 14), (33, 40, 6, 15), (256, 16, 8, 3),
              (1200, 6, 3, 83)]
GRID_CASES = [(32, 64, 12, 4, 21), (256, 256, 8, 4, 22)]     # (N, R, S, A, stream)
GRID_THR = 0.6                                               # grid_kernel's deferral threshold (capi_aux.inl)


@pytest.mark.parametrize("N,S,A,stream", POOL_CASES)
def test_fast_replay_of_pool_systems_matches_oracle(pkg, oracle, fast, N, S, A, stream):
    """The systems of the pool-sizer count test on the host: the replay, which sends a pair to the literal slow path
    where the device does (a solve that is not certified and grows past the exponent window), equals the oracle."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    e = fast.calculate(sysd)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k
    solves, fallbacks, ovf, window = e["_counts"]
    assert solves > 0 and ovf == 0, e["_counts"]
    if N == 1:
        assert fallbacks == solves


@pytest.mark.gpu
@pytest.mark.parametrize("N,S,A,stream", POOL_CASES)
def test_pool_sizer_certifies_what_the_host_replay_certifies(pkg, engine, oracle, fast, N, S, A, stream):
    """Pool sizer forced (set_option(1, 6)): candidates bit-equal to the oracle, and the device's certify_fallbacks equal
    to the host replay's count of solves it does not certify (E10 makes the solve sequence the same)."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    engine.set_option(1, 6)
    try:
        engine.load_system(sysd)
        engine.calculate()
        g = engine.candidates()
        t = engine.timing()
    finally:
        engine.set_option(1, 0)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(g[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(g[k], o[k]), k
    solves, fallbacks, ovf, window = fast.calculate(sysd)["_counts"]
    print("N = %d: %d solves, %d not certified on the host, %d on the device; %d pairs to the slow path on the host, %d "
          "on the device" % (N, solves, fallbacks, t["certify_fallbacks"], ovf + window, t["overflow_pairs"]))
    assert t["overflow_pairs"] == ovf + window
    assert t["certify_fallbacks"] == fallbacks
    if N == 1:
        assert fallbacks == solves


_grid_cache = {}


def _boundary_grid_system(pkg, fast, N, R, S, A, stream):
    """queue_system with every server's arrival rate moved (host search) to where one of its deferred levels is
    refused by the fast solve: its enclosure straddles a float32 rounding boundary."""
    key = (N, R, S, A, stream)
    if key not in _grid_cache:
        sysd = pkg.synth.queue_system(S, A, N, stream=stream, R=R)
        rng = np.random.default_rng(stream)
        arrival = sysd["srv_arrival"].copy()
        for srv in range(S):
            a = fast.boundary_arrival(sysd, srv, R, GRID_THR, float(rng.uniform(0.65, 0.95)), 400_000)
            assert a > 0, srv
            arrival[srv] = a
        sysd["srv_arrival"] = arrival
        _grid_cache[key] = sysd
    return _grid_cache[key]


def _cmp_grid(g, o):
    assert np.array_equal(g["ok"], o["ok"]) and np.array_equal(g["frontier"], o["frontier"])
    for k in ("ttft", "itl", "rho", "tput"):
        assert _bit_equal(g[k], o[k]), k


@pytest.mark.parametrize("N,R,S,A,stream", GRID_CASES)
def test_grid_deferred_replay_matches_oracle(pkg, oracle, fast, N, R, S, A, stream):
    """The host replay of the deferred grid (the same total_rate / r / 1000 lambda, analyze_admits and ratio > 0.6 rule;
    fast solve with the exact fallback on deferred levels) equals oracle.analyze_grid bit for bit, on the systems whose
    arrival rates put deferred levels next to float32 boundaries; and it does meet refusals there."""
    sysd = _boundary_grid_system(pkg, fast, N, R, S, A, stream)
    e = fast.grid(sysd, R, GRID_THR)
    _cmp_grid(e, oracle.analyze_grid(sysd, R))
    levels, deferred, refused, ovf = e["_counts"]
    print("N = %d: %d levels, %d deferred, %d of them not certified" % (N, levels, deferred, refused))
    assert ovf == 0 and refused > 0
    assert deferred <= S * A * 16 + 1024       # the device's list holds them all (capi_aux.inl)
    _cmp_grid(fast.grid(sysd, R, 0.0), oracle.analyze_grid(sysd, R))


@pytest.mark.gpu
@pytest.mark.parametrize("N,R,S,A,stream", GRID_CASES)
def test_grid_deferred_pass_refuses_what_the_host_replay_refuses(pkg, engine, oracle, fast, N, R, S, A, stream):
    """Deferral forced (set_option(6, 2)) on the boundary systems: outputs bit-equal to the oracle, and the device's
    certify_fallbacks equal to the replay's count of deferred levels not certified, which is > 0: the device's refusal
    path ran on these inputs."""
    sysd = _boundary_grid_system(pkg, fast, N, R, S, A, stream)
    engine.set_option(6, 2)
    try:
        engine.load_system(sysd)
        g = engine.analyze_grid(R)
        t = engine.timing()
    finally:
        engine.set_option(6, 0)
    _cmp_grid(g, oracle.analyze_grid(sysd, R))
    levels, deferred, refused, ovf = fast.grid(sysd, R, GRID_THR)["_counts"]
    print("N = %d: %d deferred levels, %d not certified on the host, %d on the device" %
          (N, deferred, refused, t["certify_fallbacks"]))
    assert t["overflow_pairs"] == 0 and ovf == 0
    assert t["certify_fallbacks"] == refused > 0
