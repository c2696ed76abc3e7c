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
        counts = (C.c_int64 * 3)()
        lib.emul_calculate_fast(C.byref(st), C.byref(cst), counts)
        cand["_counts"] = list(counts)
        return cand

    lib.check, lib.boundary, lib.calculate = check, boundary, calculate
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
    solves, fallbacks, ovf = e["_counts"]
    assert ovf == 0 and solves > 0
    if N >= 2:
        assert fallbacks <= 0.05 * solves, (solves, fallbacks)
