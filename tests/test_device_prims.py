"""The chain solvers' division shortcuts on the H100, against the device's IEEE division, over every float32 divisor.

Every float32 output of the sizers and the replica grid rests on (E1) (DESIGN.md §3): div_f32den(x, mu, rcp_f32den(m, mu))
is the correctly rounded x / mu.  The host build checks it with a correctly rounded seed; on the device the seed is
rcp.approx.ftz.f32, which is approximate and flushes subnormal inputs and results.  tests/device_prims/prims.cu calls the
product's own primitives (wva_core.cuh, lockstep_solve.cuh, saturation_kernel.cuh), built with the product's flags.
Divisors are split into four classes: subnormal, [2^-126, 2^126] (the E1 divisors), (2^126, 2^128) and +inf.
Measured on an H100 80GB HBM3 (400 W): the seed is within 1 ulp of 1/mu on the E1 divisors and flushes on every other
finite divisor; the largest residual |1 - mu r| there is 2^-46.56."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.test_host_logic import SEED_MAX_ULP

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASSES = ("subnormal", "e1", "high", "inf")
N_CLASS = {"subnormal": 0x007FFFFF, "e1": 0x7E800000 - 0x00800000 + 1, "high": 0x7F800000 - 0x7E800001, "inf": 1}
NX = 6                                               # dividends per divisor in prims.cu


class PrimRes(C.Structure):
    _fields_ = [("n", C.c_uint64), ("fail", C.c_uint64), ("flagged", C.c_uint64), ("skipped", C.c_uint64),
                ("max_bits", C.c_uint64), ("first", (C.c_uint64 * 2) * 16), ("lo", C.c_uint32), ("hi", C.c_uint32)]


def _f64(bits):
    return float(np.array([bits], np.uint64).view(np.float64)[0])


@pytest.fixture(scope="module")
def prims(pkg, tmp_path_factory):
    """tests/device_prims/prims.cu built with build.sh's code generation flags into a temporary directory."""
    so = str(tmp_path_factory.mktemp("device_prims") / "libprims.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "--fmad=false", "-std=c++17",
                    "-Xcompiler", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "device_prims", "prims.cu"),
                    "-lcudart"], check=True)
    lib = C.CDLL(so)
    assert lib.prims_res_size() == C.sizeof(PrimRes)
    cache = {}

    def run(name, n_res=4, *args):
        if (name, args) not in cache:
            res = (PrimRes * n_res)()
            assert getattr(lib, "prims_" + name)(res, *[C.c_uint64(a) for a in args]) == 0, "CUDA error in prims_" + name
            cache[(name, args)] = res
        return cache[(name, args)]

    lib.run = run
    lib.prims_anchor.argtypes = [C.c_void_p] * 3 + [C.c_uint64]
    return lib


def _first(r):
    return [(hex(int(r.first[k][0])), hex(int(r.first[k][1]))) for k in range(min(16, int(r.fail)))]


def test_seed_distance_and_flush_range(prims):
    """Check 1: the seed f_rcp_approx(m) against __frcp_rn(m) for every positive float32.  On the E1 divisors both are
    normal and at most SEED_MAX_ULP apart (the host E1 checks refine every seed that close); it flushes nowhere there.
    Outside, it flushes: that is why those divisors are not E1 divisors."""
    res = prims.run("seed")
    for c, name in enumerate(CLASSES):
        r = res[c]
        flush = (hex(r.lo), hex(r.hi)) if r.flagged else None
        print(f"{name}: {r.n} divisors, largest seed distance {r.max_bits} ulp, {r.flagged} flushed {flush}")
        assert r.n == N_CLASS[name]
    e1 = res[1]
    assert e1.max_bits <= SEED_MAX_ULP and e1.flagged == 0
    assert res[0].flagged == N_CLASS["subnormal"] and res[2].flagged == N_CLASS["high"]


@pytest.mark.parametrize("cls", CLASSES)
def test_reciprocal_residual(prims, cls):
    """Check 2: for every float32 divisor the solvers refine a reciprocal of (e1_divisor), r = rcp_f32den(m, mu) has
    the exact residual |1 - mu r| <= 2^-40 that E1 needs, and step_div's q0 condition |1 - mu r| + 3u <= 2^-39.99
    holds.  The other divisors are not refined: the solvers divide by them with the IEEE division."""
    c = CLASSES.index(cls)
    r = prims.run("rcp")[c]
    mx = _f64(r.max_bits)
    print(f"{cls}: {r.n} reciprocals, {r.skipped} divisors left to the IEEE division, largest residual "
          f"{mx:.3e} = 2^{np.log2(mx) if mx > 0 else float('-inf'):.2f}; first failures {_first(r)}")
    assert r.n + r.skipped == N_CLASS[cls]
    assert r.fail == 0 and r.flagged == 0
    if cls == "e1":
        assert r.skipped == 0 and mx <= 2.0 ** -40


@pytest.mark.parametrize("cls", CLASSES)
def test_div_f32den_matches_ieee_division(prims, cls):
    """Check 3a: the solvers' quotient x / mu — div_f32den with rcp_f32den for E1 divisors, d_div otherwise — equals
    __ddiv_rn bit for bit for every positive float32 mu and six x over the E3 window (both edges, all-ones significands,
    two random)."""
    c = CLASSES.index(cls)
    r = prims.run("div")[c]
    print(f"{cls}: {r.n} quotients, {r.flagged} through E1, {r.fail} wrong; first (mu, x) {_first(r)}")
    assert r.n == NX * N_CLASS[cls]
    assert r.fail == 0, _first(r)
    assert r.flagged == (r.n if cls == "e1" else 0)


@pytest.mark.parametrize("cls", CLASSES)
def test_step_div_matches_ieee_division(prims, cls):
    """Check 3b: step_div (the 3-deep E1 of the lock-step and fast solvers, q0 = p RN(lambda r)) equals
    __ddiv_rn(RN(p lambda), mu) bit for bit, and tracks the exponent of x, for every E1 divisor and six (p, lambda)
    pairs with x over the E3 window.  Pairs with another divisor never reach step_div."""
    c = CLASSES.index(cls)
    r = prims.run("step")[c]
    print(f"{cls}: {r.n} quotients, {r.flagged} left to the per-lane chain, {r.fail} wrong; first (mu, p) {_first(r)}")
    assert r.fail == 0, _first(r)
    assert r.n + r.flagged == NX * N_CLASS[cls]
    assert r.n == (NX * N_CLASS[cls] if cls == "e1" else 0)


def test_div_markstein2_matches_ieee_division(prims):
    """Check 3c: div_markstein2 (E2, the normalising division with y53 = __drcp_rn(y)) on 10^8 random pairs in the
    window, 1/8 of the divisors with all-ones significands or powers of two."""
    r = prims.run("markstein", 1, 100_000_000, 7)[0]
    assert r.n == 100_000_000
    assert r.fail == 0, _first(r)


def test_div_small_int_matches_ieee_division(prims):
    """Check 3d: div_small_int (the saturation analyser's x / n) for every n in [1, 2^24) with a random x, x = 0 and
    x = n - 1."""
    r = prims.run("small_int", 1, 11)[0]
    assert r.n == 3 * ((1 << 24) - 1)
    assert r.fail == 0, _first(r)


def test_device_division_is_ieee(prims):
    """Anchor: 10^6 of the device's __ddiv_rn results, the reference of every check above, equal numpy's IEEE float64
    division bit for bit (random operands over the whole exponent range and subnormals; a quarter of the divisors with
    24-bit significands)."""
    rng = np.random.default_rng(5)
    n = 1_000_000
    bits = rng.integers(0, 1 << 63, size=(2, n), dtype=np.uint64)      # positive, any exponent
    x, y = bits.view(np.float64)
    x, y = x.copy(), y.copy()
    y[::4] = rng.uniform(-1, 1, n // 4).astype(np.float32).astype(np.float64) * 2.0 ** rng.integers(-149, 128, n // 4)
    ok = np.isfinite(x) & np.isfinite(y) & (y != 0)
    x, y = np.ascontiguousarray(x[ok]), np.ascontiguousarray(y[ok])
    q = np.empty_like(x)
    assert prims.prims_anchor(x.ctypes.data, y.ctypes.data, q.ctypes.data, len(x)) == 0
    with np.errstate(all="ignore"):
        ref = x / y
    assert len(x) > 0.99 * n
    assert np.array_equal(q.view(np.uint64), ref.view(np.uint64)), np.flatnonzero(q.view(np.uint64) != ref.view(np.uint64))[:8]
