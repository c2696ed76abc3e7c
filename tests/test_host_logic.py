"""CPU-side tests (no GPU): the host build of the device core vs the oracle, the C-ABI library's exported
symbols, the ctypes struct images, the synthetic generators and the model-sharding plumbing."""
import ctypes as C
import importlib
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# Largest distance, in float32 ulps, of the device's reciprocal seed rcp.approx.ftz.f32 from the correctly rounded 1/mu
# over the (E1) divisors [2^-126, 2^126]; test_device_prims.py measures it over every float32 on the H100.
SEED_MAX_ULP = 1
F32_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_arrv_rate")


@pytest.fixture(scope="session")
def emul(pkg):
    """tests/host_emul/libemul.so: csrc/wva_core.cuh compiled for the host (test infrastructure)."""
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "host_emul")], check=True)
    lib = C.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    abi = pkg._abi
    lib.emul_calculate.argtypes = [C.POINTER(abi.System), C.POINTER(abi.Candidates)] + [C.POINTER(C.c_int64)] * 3
    lib.emul_check_div_f32den.restype = C.c_int64
    lib.emul_check_div_f32den.argtypes = [C.c_int64, C.c_uint64, C.c_int]
    lib.emul_check_step_div.restype = C.c_int64
    lib.emul_check_step_div.argtypes = [C.c_int64, C.c_uint64, C.c_int]
    lib.emul_check_e1_range.restype = C.c_int64
    lib.emul_check_seed_ftz.restype = C.c_int64
    lib.emul_check_div_markstein2.restype = C.c_int64
    lib.emul_check_div_markstein2.argtypes = [C.c_int64, C.c_uint64]

    def calculate(sysd):
        st, keep = abi.make_system(sysd)
        cst, cand = abi.alloc_candidates(st.n_servers, st.n_acc)
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        lib.emul_calculate(C.byref(st), C.byref(cst), C.byref(a), C.byref(b), C.byref(c))
        cand["_solves"], cand["_states"], cand["_overflow"] = a.value, b.value, c.value
        return cand

    lib.emul_calculate_spec.argtypes = [C.POINTER(abi.System), C.POINTER(abi.Candidates)]

    def calculate_spec(sysd):
        st, keep = abi.make_system(sysd)
        cst, cand = abi.alloc_candidates(st.n_servers, st.n_acc)
        lib.emul_calculate_spec(C.byref(st), C.byref(cst))
        return cand

    lib.emul_calculate_dual.argtypes = [C.POINTER(abi.System), C.POINTER(abi.Candidates)]

    def calculate_dual(sysd):
        st, keep = abi.make_system(sysd)
        cst, cand = abi.alloc_candidates(st.n_servers, st.n_acc)
        lib.emul_calculate_dual(C.byref(st), C.byref(cst))
        return cand

    lib.emul_calculate_spec2.argtypes = [C.POINTER(abi.System), C.POINTER(abi.Candidates), C.POINTER(C.c_int64)]

    def calculate_spec2(sysd):
        st, keep = abi.make_system(sysd)
        cst, cand = abi.alloc_candidates(st.n_servers, st.n_acc)
        stats = (C.c_int64 * 4)()
        lib.emul_calculate_spec2(C.byref(st), C.byref(cst), stats)
        cand["_stats"] = list(stats)
        return cand

    lib.calculate_spec2 = calculate_spec2
    lib.calculate = calculate
    lib.calculate_dual = calculate_dual
    lib.calculate_spec = calculate_spec
    return lib


def _bit_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def test_exact_division_tricks(emul):
    """(E1)/(E2) of csrc/wva_core.cuh against the IEEE operator, incl. all-ones / power-of-two divisors.  The E1 checks
    draw divisors from every exponent of [2^-126, 2^126] and refine every seed within SEED_MAX_ULP of RN(1/mu), the
    seeds the device's rcp.approx.ftz.f32 can return there."""
    assert emul.emul_check_div_f32den(2_000_000, 1, SEED_MAX_ULP) == 0
    assert emul.emul_check_div_markstein2(5_000_000, 2) == 0
    assert emul.emul_check_step_div(2_000_000, 3, SEED_MAX_ULP) == 0


def test_e1_divisor_range_and_host_seed_flush(emul):
    """e1_divisor is true exactly on [2^-126, 2^126] over all 2^32 float32 bit patterns, and the host seed flushes like
    rcp.approx.ftz.f32: a subnormal mu reads as 0 (seed inf), a subnormal 1/mu is returned as 0."""
    assert emul.emul_check_e1_range() == 0
    assert emul.emul_check_seed_ftz() == 0


@pytest.mark.parametrize("S,A,N,stream", [(10, 4, 32, 1), (40, 8, 16, 7), (12, 6, 128, 2), (4, 4, 256, 3),
                                          (20, 3, 1, 11), (16, 3, 5, 12)])
def test_lane_state_machine_matches_oracle(pkg, oracle, emul, S, A, N, stream):
    """The flattened sizer lane (early exits, two-pass chain, shared bisection endpoints) reproduces
    CreateAllocation bit for bit."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    e = emul.calculate(sysd)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k
    assert e["_overflow"] == 0 and e["_solves"] <= o["_solves"]


@pytest.mark.parametrize("S,A,N,stream", [(10, 4, 32, 1), (40, 8, 16, 7), (10, 6, 128, 2), (20, 3, 1, 11)])
def test_speculative_bisection_matches_oracle(pkg, oracle, emul, S, A, N, stream):
    """The tree-speculative search of the warp-per-pair sizer takes exactly BinarySearch's branches."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    e = emul.calculate_spec(sysd)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k


@pytest.mark.parametrize("S,A,N,stream", [(10, 4, 32, 1), (40, 8, 16, 7), (10, 6, 128, 2), (20, 3, 1, 11)])
def test_dual_chain_driver_matches_oracle(pkg, oracle, emul, S, A, N, stream):
    """TTFT and ITL searches advanced in the same round (lock-step lane sizer) = the sequential searches."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    sysd["srv_slo_itl"][::5] = 0.0       # TTFT-only servers
    sysd["srv_slo_ttft"][1::5] = 0.0     # ITL-only servers
    e = emul.calculate_dual(sysd)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k


@pytest.mark.parametrize("S,A,N,stream", [(10, 4, 32, 1), (40, 8, 16, 7), (10, 6, 128, 2), (20, 3, 1, 11), (16, 3, 5, 12)])
def test_speculative_split_driver_matches_oracle(pkg, oracle, emul, S, A, N, stream):
    """One search per item, the second chain on the predicted next bisection point (spec2_*): a wrong guess must
    never change a decision, a right one must be consumed exactly as BinarySearch would have evaluated it."""
    sysd = pkg.synth.queue_system(S, A, N, stream=stream)
    sysd["srv_slo_itl"][::5] = 0.0       # TTFT-only servers
    sysd["srv_slo_ttft"][1::5] = 0.0     # ITL-only servers
    e = emul.calculate_spec2(sysd)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k
    rounds, steps, spec_rounds, hits = e["_stats"]
    if N >= 16:
        assert steps > 1.3 * rounds, (rounds, steps, spec_rounds, hits)   # the guesses do pay


def test_overflow_rescale_path_matches_oracle(pkg, oracle, emul):
    sysd = pkg.synth.queue_system(2, 2, 1024, stream=31)
    sysd["perf_alpha"][:] = 4.0; sysd["perf_beta"][:] = 0.0; sysd["perf_gamma"][:] = 0.0
    sysd["srv_in_tokens"][:] = 0; sysd["srv_out_tokens"][:] = 16; sysd["perf_at_tokens"][:] = 16
    sysd["srv_arrival"][:] = 60.0 * 2000
    sysd["srv_slo_ttft"][:] = 5000.0; sysd["srv_slo_itl"][:] = 0.0
    e = emul.calculate(sysd)
    o = oracle.calculate(sysd)
    assert e["_overflow"] > 0
    for k in ("state", "num_replicas", "batch_size"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k
    assert (o["state"] == 1).any()


def test_subnormal_tail_matches_oracle(pkg, oracle, emul):
    """Tiny arrival rates drive p~ through the subnormal range (gradual underflow must be kept, SURVEY H4)."""
    sysd = pkg.synth.queue_system(6, 3, 64, stream=13)
    sysd["srv_arrival"][:] = np.float32(1e-3)
    sysd["srv_slo_ttft"][:] = 1e6; sysd["srv_slo_itl"][:] = 1e6
    e = emul.calculate(sysd)
    o = oracle.calculate(sysd)
    for k in ("state", "num_replicas"):
        assert np.array_equal(e[k], o[k]), k
    for k in F32_FIELDS:
        assert _bit_equal(e[k], o[k]), k


# ---- the C-ABI library -----------------------------------------------------------------------------------
def _declared_functions():
    src = open(os.path.join(ROOT, "include", "wva_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(wva_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(pkg):
    lib_path = pkg.lib_path()
    assert os.path.exists(lib_path), "csrc/libwva_b200.so missing: run __graft_entry__.build()"
    lib = C.CDLL(lib_path)
    declared = _declared_functions()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/wva_b200.h but not exported"
    assert sorted(pkg.engine.EXPORTS) == declared


def test_no_gpu_means_loud_failure(pkg):
    """No CPU fallback: without a CUDA device the product refuses to construct (no compute calls made)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(pkg.WvaError):
        pkg.Engine(device=0)


def test_product_never_touches_oracle():
    """The package must not import, link or dlopen anything under oracle/ or tests/."""
    pkg_dir = os.path.join(ROOT, "llm-d-workload-variant-autoscaler_b200")
    for dirpath, _, files in os.walk(pkg_dir):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".inl", ".h", ".sh", ".cpp", ".hpp", ".go")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "liboracle" not in txt and "libemul" not in txt, (dirpath, f)
                assert not re.search(r"^\s*(from|import)\s+[^\n]*(oracle|host_emul)", txt, flags=re.M), (dirpath, f)
                assert not re.search(r'#include\s+"[^"]*(oracle|host_emul)/', txt), (dirpath, f)


def test_struct_images_match_header(pkg):
    """ctypes struct sizes vs sizeof() from the C header (compiled with the host compiler)."""
    code = r'''
#include <stdio.h>
#include "wva_b200.h"
int main(){printf("%zu %zu %zu %zu %zu %zu\n", sizeof(wva_system), sizeof(wva_candidates), sizeof(wva_solution),
 sizeof(wva_timing), sizeof(wva_saturation_in), sizeof(wva_saturation_out));return 0;}
'''
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        open(os.path.join(td, "s.c"), "w").write(code)
        subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(td, "s"),
                        os.path.join(td, "s.c")], check=True)
        out = subprocess.run([os.path.join(td, "s")], capture_output=True, text=True, check=True).stdout.split()
    abi = pkg._abi
    got = [C.sizeof(x) for x in (abi.System, abi.Candidates, abi.Solution, abi.Timing, abi.SaturationIn,
                                 abi.SaturationOut)]
    assert got == [int(x) for x in out]


# ---- generators and sharding ------------------------------------------------------------------------------------
def test_synth_is_deterministic(pkg):
    a = pkg.synth.baseline_config(2, scale=0.01)
    b = pkg.synth.baseline_config(2, scale=0.01)
    for k, v in a.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(v, b[k]), k
    assert a["n_servers"] == 10 and a["n_acc"] == 16


def test_model_sharding_is_a_partition(pkg, oracle):
    """Sharded by server index (s % world == rank): shard results concatenate to the unsharded result and the
    by-type partials sum to the global ones — the invariant the multi-GPU path relies on."""
    d = pkg.synth.queue_system(30, 4, 16, stream=15)
    full = oracle.calculate(d)
    fsol = oracle.solve(d, full)
    world = 4
    tc = np.zeros_like(fsol["type_count"])
    seen = np.zeros(30, bool)
    for rank in range(world):
        sd, idx = pkg.synth.shard_system(d, rank, world)
        c = oracle.calculate(sd)
        s = oracle.solve(sd, c)
        assert np.array_equal(c["num_replicas"], full["num_replicas"][idx])
        assert _bit_equal(c["value"], full["value"][idx])
        assert np.array_equal(s["acc"], fsol["acc"][idx])
        tc += s["type_count"]
        seen[idx] = True
    assert seen.all() and np.array_equal(tc, fsol["type_count"])


@pytest.mark.parametrize("threads", [1, 2, 3, 8, 64])
def test_ingest_scatter_threads_equal_the_serial_map_assignment(emul, threads):
    """csrc/ingest_scatter.hpp (the host side of wva_ingest_write): split over threads by slot range, a response in any
    order with duplicate samples, unknown pods (slot < 0) and every slot residue gives exactly what the reference's map
    assignment gives — the LAST sample of a pod wins (internal/collector/replica_metrics.go:133-160)."""
    g = np.random.default_rng(77 + threads)
    S, n = 10_007, 60_000                                   # every slot reported ~6 times: duplicates everywhere
    slot = g.integers(-3, S, n).astype(np.int32)
    value = g.random(n)
    col = np.full(S, -1.0); has = np.zeros(S, np.uint8)
    has[::5] = 2                                            # bits of the other vector stay
    want_col, want_has = col.copy(), has.copy()
    for k, v in zip(slot.tolist(), value.tolist()):         # the serial map assignment
        if k >= 0:
            want_col[k] = v; want_has[k] |= 1
    f = emul.emul_ingest_scatter
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    assert f(col.ctypes.data, has.ctypes.data, S, 1, n, slot.ctypes.data, value.ctypes.data, threads) == 0
    assert np.array_equal(col, want_col) and np.array_equal(has, want_has)
    # a slot past the registry is an argument error, whichever range it falls behind
    slot[n // 2] = S + 5
    assert f(col.ctypes.data, has.ctypes.data, S, 1, n, slot.ctypes.data, value.ctypes.data, threads) == 1
    # tiny registries: fewer 64-slot blocks than threads
    col2 = np.zeros(3); has2 = np.zeros(3, np.uint8)
    s2 = np.array([2, 0, 2, -1], np.int32); v2 = np.array([1.0, 2.0, 3.0, 4.0])
    assert f(col2.ctypes.data, has2.ctypes.data, 3, 2, 4, s2.ctypes.data, v2.ctypes.data, threads) == 0
    assert col2.tolist() == [2.0, 0.0, 3.0] and has2.tolist() == [2, 0, 2]


@pytest.mark.parametrize("order", ["registry", "shuffled", "mostly_sorted_with_duplicates"])
def test_ingest_scatter_auto_mode(emul, order):
    """threads = 0: the library chooses — the serial loop for a response in registry order, the partition otherwise."""
    g = np.random.default_rng(5)
    S = 70_001
    slot = np.arange(S, dtype=np.int32)
    if order == "shuffled":
        slot = g.permutation(S).astype(np.int32)
    elif order == "mostly_sorted_with_duplicates":
        slot = np.concatenate([slot, g.integers(0, S, 3000).astype(np.int32)])
    n = slot.size
    value = g.random(n)
    want = np.zeros(S); want[slot] = value                   # numpy assigns in order: the last duplicate wins
    col = np.zeros(S); has = np.zeros(S, np.uint8)
    f = emul.emul_ingest_scatter
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    assert f(col.ctypes.data, has.ctypes.data, S, 2, n, slot.ctypes.data, value.ctypes.data, 0) == 0
    assert np.array_equal(col, want) and (has == 2).all()
