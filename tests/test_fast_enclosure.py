"""The error bounds of the certified fast solve (DESIGN.md §3, E12) against exact arithmetic.

fast_solve_finish accepts a solve when v +- 4(a + b) rounds to one float32 for L, Lserv and 1 - p[K], where (a) bounds
how far the reference's float64 values are from the exact ones and (b) how far the fast path's own values are.  The
end-to-end tests in test_fast_solve.py rarely meet a value near a rounding boundary, so a bound that is too small would
pass them.  Here every bound is checked directly: the host build of the fast solve reports its values and bounds through
WVA_FAST_PROBE (empty in the product), and tests/host_emul/enclosure_emul.cpp compares them with a binary128 chain over
all K + 1 states (the exact values) and with a literal float64 chain in the reference's loop order."""
import concurrent.futures as cf
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REGIMES = ("random", "lambda_max", "omega_floor", "light", "non_monotone", "heavy_pK")
N_VALUES = (2, 3, 7, 16, 17, 18, 33, 256, 1200)    # the head chunk (WVA_TILE_CHUNK = 16) edges: N - 1 below, at, above
VALUES = ("L", "Lserv", "pK")
THREADS = max(1, min(8, os.cpu_count() or 1))


@pytest.fixture(scope="module")
def enc(tmp_path_factory):
    """tests/host_emul/enclosure_emul.cpp (fast_emul.cpp with the probe and the exact chains), built into a temporary
    directory."""
    src = os.path.join(ROOT, "tests", "host_emul", "enclosure_emul.cpp")
    so = str(tmp_path_factory.mktemp("enclosure_emul") / "libencemul.so")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-pthread",
                    "-shared", "-o", so, src], check=True)
    lib = C.CDLL(so)
    lib.enc_cell.argtypes = [C.c_int, C.c_int, C.c_int64, C.c_uint64, C.POINTER(C.c_double)]
    lib.enc_exact.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.c_float, C.POINTER(C.c_double)]
    lib.enc_boundary.argtypes = [C.c_int, C.c_int64, C.c_int, C.c_uint64, C.c_double, C.POINTER(C.c_int64)]
    return lib


def _cell(lib, rg, N, n, seed):
    out = (C.c_double * 21)()
    lib.enc_cell(rg, N, n, seed, out)
    o = list(out)
    return {"draws": int(o[0]), "probed": int(o[1]), "cert": int(o[2]), "exited": int(o[3]),
            "ratio_a": o[4:7], "ratio_b": o[7:10], "viol_a": [int(v) for v in o[10:13]],
            "viol_b": [int(v) for v in o[13:16]], "literal_diff": int(o[16]), "cert_diff": int(o[17]),
            "skipped": int(o[18]), "subnormal_pK": int(o[19]), "heavy_pK": int(o[20])}


def _solves(N):
    # the binary128 chain costs ~0.2 us per state: ~2.5 ms per solve at N = 1200 (K = 13 200)
    return 40 if N == 1200 else 300 if N == 256 else 3000 if N >= 16 else 1500


def test_enclosure_bounds_hold_against_exact_arithmetic(enc):
    """Every probed solve, six regimes x N in {2, 3, 7, 16, 17, 18, 33, 256, 1200}: |ref64 - exact| <= (a) and
    |fast - exact| <= (b) for L, Lserv and p[K], before the safety factor 4, with no exception.  The literal float64
    chain's float32 statistics equal literal_solve's and the exact lane solver's, and every certified lane equals them."""
    jobs = {(rg, N): (rg, N, _solves(N), 1000 * rg + N) for rg in range(len(REGIMES)) for N in N_VALUES}
    with cf.ThreadPoolExecutor(THREADS) as ex:
        res = dict(zip(jobs, ex.map(lambda a: _cell(enc, *a), jobs.values())))
    print("\nlargest error / bound, (a) reference vs exact | (b) fast vs exact")
    print("%-13s %5s %6s | %-26s | %-26s" % ("regime", "N", "probed", "a: L  Lserv  pK", "b: L  Lserv  pK"))
    bad = []
    for (rg, N), r in sorted(res.items()):
        print("%-13s %5d %6d | %8.3g %8.3g %8.3g | %8.3g %8.3g %8.3g" %
              ((REGIMES[rg], N, r["probed"]) + tuple(r["ratio_a"]) + tuple(r["ratio_b"])))
        if any(r["viol_a"]) or any(r["viol_b"]) or r["literal_diff"] or r["cert_diff"] or r["skipped"]:
            bad.append((REGIMES[rg], N, r))
    assert not bad, bad
    for (rg, N), r in res.items():
        assert max(r["ratio_a"] + r["ratio_b"]) <= 1.0
        # every regime forms its enclosure on most of its draws (non-monotone tables at N = 1200 leave the E3 window
        # more often; heavy_pK keeps only the draws with p[K] in range and is checked below)
        if REGIMES[rg] != "heavy_pK":
            assert r["probed"] >= (0.1 if N == 1200 else 0.5) * r["draws"], (REGIMES[rg], N, r)
    # the regimes reach what they are meant to reach
    for N in N_VALUES:
        light = res[(REGIMES.index("light"), N)]
        assert (light["exited"] == light["probed"]) if N >= 18 else light["exited"] == 0, (N, light)
        heavy = res[(REGIMES.index("heavy_pK"), N)]
        assert heavy["heavy_pK"] == heavy["probed"] > 0, (N, heavy)
    # subnormal p[K] (no absolute underflow term in (b) would fail here) occurs among the random draws
    assert sum(r["subnormal_pK"] for r in res.values()) > 0


def _fraction_chain(tab, N, K, lam):
    lam = Fraction(float(lam))
    mus = [Fraction(float(t)) for t in tab]
    p, S, T, U = Fraction(1), Fraction(1), Fraction(0), Fraction(0)
    for n in range(K):
        p = p * lam / mus[min(n, N - 1)]
        S += p
        T += (n + 1) * p
        U += min(n + 1, N) * p
    return T / S, U / S, p / S


def test_binary128_chain_matches_fractions(enc):
    """The exact reference itself: 240 solves at N <= 32 (monotone and arbitrary float32 tables, lambda up to 1.2 mu)
    against stdlib Fraction arithmetic, to 2^-100 relative."""
    rng = np.random.default_rng(2026)
    worst = 0.0
    for i in range(240):
        N = int(rng.choice([2, 3, 7, 16, 32]))
        K = N + 10 * N
        tab = (rng.uniform(0.5, 4.0, N) * 2.0 ** rng.integers(-6, 6)).astype(np.float32)
        if i % 2 == 0:
            tab.sort()
        lam = np.float32(float(tab[-1]) * rng.uniform(0.01, 1.2))
        out = (C.c_double * 9)()
        enc.enc_exact(tab.ctypes.data_as(C.POINTER(C.c_float)), N, K, float(lam), out)
        for k, ex in enumerate(_fraction_chain(tab, N, K, lam)):
            got = (Fraction(out[3 * k]) + Fraction(out[3 * k + 1])) * Fraction(2) ** int(out[3 * k + 2])
            err = abs(got - ex) / ex
            worst = max(worst, float(err))
            assert err <= Fraction(1, 2 ** 100), (i, N, VALUES[k], float(err))
    print("binary128 chain vs Fraction: largest relative error %.3g (2^%.1f)" % (worst, np.log2(worst) if worst else -np.inf))


@pytest.mark.parametrize("N,models,steps", [(32, 200, 1000), (256, 200, 1000), (1200, 250, 1000)])
def test_enclosure_refuses_boundaries_at_sizing_batch_sizes(enc, N, models, steps):
    """Boundary search: consecutive float32 lambda of configs[2]-shaped models.  Solves whose reference L or Lserv lies
    within 10^-11 (relative) of a float32 midpoint, or whose f_sub(1, (float)p[K]) changes within 10^-11 of p[K], are
    certified only when bit-equal to the literal chain; none within the a-priori floor of the enclosure is certified."""
    chunks = [(N, models // THREADS + (1 if t < models % THREADS else 0), steps, 7919 * N + t) for t in range(THREADS)]

    def run(a):
        st = (C.c_int64 * 7)()
        enc.enc_boundary(*a, 1e-11, st)
        return np.array(st, dtype=np.int64)

    with cf.ThreadPoolExecutor(THREADS) as ex:
        near, cert, wrong, floor_hits, floor_cert, probed, near_pk = sum(ex.map(run, [c for c in chunks if c[1] > 0]))
    print("N = %d: %d solves probed, %d near a boundary (%d next to a change of 1 - p[K]), %d of them certified; "
          "%d within the a-priori floor" % (N, probed, near, near_pk, cert, floor_hits))
    assert near - near_pk > 50 and near_pk > 0, (near, near_pk, probed)
    assert wrong == 0, (near, cert, wrong)
    assert floor_cert == 0, (floor_hits, floor_cert)
