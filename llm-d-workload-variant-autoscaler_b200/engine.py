"""Python binding of the C-ABI (include/wva_b200.h) — the call path tests/ and bench.py use.

``Engine`` owns one ``wva_ctx`` (one GPU).  Method names mirror the reference
entry points they replace:

    load_system      System.SetFromSpec           pkg/core/system.go:82
    calculate        System.Calculate             pkg/core/system.go:258
    update_servers   AddServerInfoToSystemData    internal/utils/utils.go:204 (loads + current allocations)
    recalculate      System.Calculate, for the servers update_servers / update_server_set changed
    update_server_set  System.AddServerFromSpec / RemoveServer   pkg/core/system.go:160 (the whole server set)
    update_tables    accelerator costs + ModelAcceleratorPerfData, for the (server, accelerator) pairs that read them
    solve            Manager.Optimize             pkg/manager/manager.go:21
    candidates       Server.AllAllocations        pkg/core/server.go:138
    solution         System.GenerateSolution      pkg/core/system.go:303
    analyze_grid     QueueAnalyzer.Analyze grid   pkg/analyzer/queueanalyzer.go:127
    grid_update      the resident grid, for the servers whose load update_servers changed
    mm1k_eval        MM1KModel.Solve              pkg/analyzer/mm1kmodel.go:30
    saturation_v1    AnalyzeModelSaturation + CalculateSaturationTargets
                                                  internal/saturation/analyzer.go:31,290
    limit            DefaultLimiter.Limit         internal/engines/pipeline/default_limiter.go:42

There is no CPU fallback: a missing library or a missing GPU raises WvaError.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _abi as abi

_HERE = os.path.dirname(os.path.abspath(__file__))


class WvaError(RuntimeError):
    pass


def lib_path() -> str:
    return os.path.join(_HERE, "csrc", "libwva_b200.so")


_lib = None


def load_library():
    """dlopen csrc/libwva_b200.so (built in-tree by __graft_entry__.build()); raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise WvaError(f"{p} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU fallback)")
    L = C.CDLL(p)
    ctxp = C.c_void_p
    L.wva_create.argtypes = [C.c_int32, C.POINTER(ctxp)]
    L.wva_destroy.argtypes = [ctxp]
    L.wva_strerror.argtypes = [C.c_int32]
    L.wva_strerror.restype = C.c_char_p
    L.wva_last_error.argtypes = [ctxp]
    L.wva_last_error.restype = C.c_char_p
    L.wva_launch_count.argtypes = [ctxp]
    L.wva_launch_count.restype = C.c_int64
    L.wva_set_option.argtypes = [ctxp, C.c_int32, C.c_int32]
    L.wva_set_optimizer.argtypes = [ctxp, C.c_int32, C.c_int32, C.c_int32]
    L.wva_set_capacity.argtypes = [ctxp, C.c_void_p]
    L.wva_comm_unique_id.argtypes = [C.c_void_p]
    L.wva_comm_init_rank.argtypes = [ctxp, C.c_int32, C.c_int32, C.c_void_p]
    L.wva_comm_shard.argtypes = [ctxp, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.wva_group_create.argtypes = [C.c_void_p, C.c_int32, C.POINTER(ctxp)]
    L.wva_group_destroy.argtypes = [ctxp]
    L.wva_group_size.argtypes = [ctxp]
    L.wva_group_ctx.argtypes = [ctxp, C.c_int32]
    L.wva_group_ctx.restype = ctxp
    L.wva_group_optimize.argtypes = [ctxp, C.POINTER(abi.System), C.POINTER(abi.Solution)]
    L.wva_group_saturation_v1.argtypes = [ctxp, C.POINTER(abi.SaturationIn), C.POINTER(abi.SaturationOut)]
    L.wva_ingest_create.argtypes = [ctxp, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(ctxp),
                                    C.POINTER(abi.IngestColumns), C.POINTER(abi.IngestResults)]
    L.wva_ingest_create_decisions.argtypes = [ctxp, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                              C.POINTER(ctxp), C.POINTER(abi.IngestColumns), C.POINTER(abi.IngestResults),
                                              C.POINTER(abi.IngestDecisionColumns), C.POINTER(abi.IngestDecisionResults)]
    L.wva_ingest_destroy.argtypes = [ctxp]
    L.wva_ingest_begin.argtypes = [ctxp]
    L.wva_ingest_write.argtypes = [ctxp, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]
    L.wva_ingest_commit.argtypes = [ctxp]
    L.wva_ingest_v2_create.argtypes = [ctxp, C.c_int64, C.c_int64, C.c_int64] + [C.c_void_p] * 4 + [ctxp, C.POINTER(ctxp),
                                       C.POINTER(abi.IngestV2Columns), C.POINTER(abi.IngestV2Results)]
    L.wva_ingest_v2_destroy.argtypes = [ctxp]
    L.wva_ingest_v2_begin.argtypes = [ctxp]
    L.wva_ingest_v2_write.argtypes = [ctxp, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]
    L.wva_ingest_v2_write_cache_config.argtypes = [ctxp, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    L.wva_ingest_v2_analyze.argtypes = [ctxp]
    L.wva_ingest_v2_decide.argtypes = [ctxp]
    L.wva_load_system.argtypes = [ctxp, C.POINTER(abi.System)]
    L.wva_calculate.argtypes = [ctxp]
    L.wva_update_servers.argtypes = [ctxp] + [C.c_void_p] * len(abi.CYCLE_ARRAYS)
    L.wva_recalculate.argtypes = [ctxp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.wva_update_server_set.argtypes = [ctxp, C.c_int32, C.c_void_p, C.POINTER(abi.System)]
    L.wva_update_tables.argtypes = [ctxp, C.POINTER(abi.System), C.POINTER(C.c_int64)]
    L.wva_solve.argtypes = [ctxp]
    L.wva_get_candidates.argtypes = [ctxp, C.POINTER(abi.Candidates)]
    L.wva_set_candidates.argtypes = [ctxp, C.POINTER(abi.Candidates)]
    L.wva_get_solution.argtypes = [ctxp, C.POINTER(abi.Solution)]
    L.wva_analyze_grid.argtypes = [ctxp, C.c_int32] + [C.c_void_p] * 6
    L.wva_grid_run.argtypes = [ctxp, C.c_int32, C.c_int32]
    L.wva_grid_fetch.argtypes = [ctxp] + [C.c_void_p] * 6
    L.wva_grid_update.argtypes = [ctxp, C.POINTER(C.c_int64)]
    L.wva_saturation_upload.argtypes = [ctxp, C.POINTER(abi.SaturationIn)]
    L.wva_saturation_run.argtypes = [ctxp, C.c_int32]
    L.wva_saturation_fetch.argtypes = [ctxp, C.POINTER(abi.SaturationOut)]
    L.wva_mm1k_eval.argtypes = [ctxp, C.c_int64] + [C.c_void_p] * 11
    L.wva_saturation_v1.argtypes = [ctxp, C.POINTER(abi.SaturationIn), C.POINTER(abi.SaturationOut)]
    L.wva_limit.argtypes = [ctxp, C.c_int64, C.c_int32] + [C.c_void_p] * 10
    L.wva_saturation_v2.argtypes = [ctxp, C.POINTER(abi.SaturationV2In), C.POINTER(abi.SaturationV2Out)]
    L.wva_cost_aware_optimize.argtypes = [ctxp, C.c_int64, C.c_int64] + [C.c_void_p] * 8
    L.wva_enforce.argtypes = [ctxp, C.c_int64, C.c_int64] + [C.c_void_p] * 8
    L.wva_pipeline_v2.argtypes = [ctxp, C.POINTER(abi.SaturationV2In)] + [C.c_void_p] * 5 + [C.POINTER(abi.SaturationV2Out), C.c_void_p, C.c_void_p]
    L.wva_k2_history_create.argtypes = [ctxp, C.c_int64, C.c_int64, C.c_int64] + [C.c_void_p] * 4 + [C.POINTER(ctxp)]
    L.wva_k2_history_destroy.argtypes = [ctxp]
    L.wva_k2_history_keys.argtypes = [ctxp]
    L.wva_k2_history_keys.restype = C.c_int64
    L.wva_k2_resolve.argtypes = [ctxp, C.POINTER(abi.K2In), C.POINTER(abi.K2Out)]
    L.wva_k2_history_export.argtypes = [ctxp] + [C.c_void_p] * 5
    L.wva_k2_history_import.argtypes = [ctxp, C.c_int64] + [C.c_void_p] * 5
    L.wva_host_alloc.argtypes = [C.c_size_t, C.POINTER(C.c_void_p)]
    L.wva_host_free.argtypes = [C.c_void_p]
    L.wva_last_timing.argtypes = [ctxp, C.POINTER(abi.Timing)]
    L.wva_microbench_fp64.argtypes = [ctxp, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    _lib = L
    return L


EXPORTS = ["wva_set_option", "wva_create", "wva_destroy", "wva_strerror", "wva_last_error", "wva_launch_count",
           "wva_load_system", "wva_calculate", "wva_update_servers", "wva_recalculate", "wva_update_server_set", "wva_update_tables", "wva_solve", "wva_get_candidates", "wva_set_candidates", "wva_get_solution",
           "wva_analyze_grid", "wva_grid_run", "wva_grid_fetch", "wva_grid_update", "wva_mm1k_eval", "wva_saturation_v1",
           "wva_saturation_upload", "wva_saturation_run", "wva_saturation_fetch", "wva_limit", "wva_saturation_v2",
           "wva_cost_aware_optimize", "wva_enforce", "wva_pipeline_v2", "wva_host_alloc", "wva_host_free", "wva_last_timing",
           "wva_microbench_fp64", "wva_set_optimizer", "wva_set_capacity", "wva_comm_unique_id", "wva_comm_init_rank",
           "wva_comm_shard", "wva_group_create", "wva_group_destroy", "wva_group_size", "wva_group_ctx",
           "wva_group_optimize", "wva_group_saturation_v1", "wva_ingest_create", "wva_ingest_destroy", "wva_ingest_begin",
           "wva_ingest_write", "wva_ingest_commit", "wva_ingest_create_decisions", "wva_k2_history_create",
           "wva_k2_history_destroy", "wva_k2_history_keys", "wva_k2_resolve", "wva_k2_history_export",
           "wva_k2_history_import", "wva_ingest_v2_create", "wva_ingest_v2_destroy", "wva_ingest_v2_begin",
           "wva_ingest_v2_write", "wva_ingest_v2_write_cache_config", "wva_ingest_v2_analyze", "wva_ingest_v2_decide"]


def comm_unique_id() -> bytes:
    """128-byte NCCL id for wva_comm_init_rank: made on ONE rank, carried to the others by the host."""
    lib = load_library()
    buf = (C.c_uint8 * 128)()
    rc = lib.wva_comm_unique_id(buf)
    if rc != abi.WVA_OK:
        raise WvaError(f"wva_comm_unique_id: {lib.wva_strerror(rc).decode()}")
    return bytes(buf)


def pinned_empty(shape, dtype) -> np.ndarray:
    """numpy array in page-locked host memory (wva_host_alloc): uploads from it and fetches into it are DMA at link
    speed.  The memory is released when the array (and every view of it) is garbage collected."""
    import weakref
    lib = load_library()
    dt = np.dtype(dtype)
    n = int(np.prod(shape)) if np.ndim(shape) else int(shape)
    nbytes = max(n * dt.itemsize, 1)
    p = C.c_void_p()
    rc = lib.wva_host_alloc(nbytes, C.byref(p))
    if rc != abi.WVA_OK or not p.value:
        raise WvaError(f"wva_host_alloc({nbytes}) failed: {lib.wva_strerror(rc).decode()}")
    buf = (C.c_uint8 * nbytes).from_address(p.value)
    weakref.finalize(buf, lib.wva_host_free, C.c_void_p(p.value))
    return np.frombuffer(buf, dtype=dt, count=n).reshape(shape)


def pinned_copy(d: dict) -> dict:
    """the same batch / system dict with every ndarray moved into page-locked memory"""
    out = {}
    for k, v in d.items():
        if isinstance(v, np.ndarray) and v.size:
            a = pinned_empty(v.shape, v.dtype)
            a[...] = v
            out[k] = a
        else:
            out[k] = v
    return out


class Engine:
    def __init__(self, device: int = 0):
        self.lib = load_library()
        self.ctx = C.c_void_p()
        rc = self.lib.wva_create(device, C.byref(self.ctx))
        if rc != abi.WVA_OK:
            self.ctx = None
            raise WvaError(f"wva_create(device={device}) failed: {self.lib.wva_strerror(rc).decode()}")
        self.S = self.A = self.T = 0
        self.lo = self.hi = 0          # block of servers this context sizes (the whole system without a communicator)
        self.world, self.rank = 1, 0
        self._grid_R = 0               # R of the resident grid (grid_run / analyze_grid)
        # optional allocator (name, n, dtype) -> 1-D array for the result buffers of saturation_fetch() and limit(),
        # e.g. views of page-locked buffers from pinned_empty() that the caller reuses from batch to batch
        self.host_alloc = None

    def _check(self, rc, what):
        if rc != abi.WVA_OK:
            detail = self.lib.wva_last_error(self.ctx).decode()
            raise WvaError(f"{what}: {self.lib.wva_strerror(rc).decode()} {detail}")

    def close(self):
        if self.ctx:
            self.lib.wva_destroy(self.ctx)
            self.ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_option(self, option: int, value: int):
        self._check(self.lib.wva_set_option(self.ctx, option, value), "wva_set_option")

    # ---- multi-GPU ----------------------------------------------------------------------------
    def comm_init(self, world: int, rank: int, unique_id: bytes):
        """Join the NCCL communicator of `world` contexts (before load_system).  From then on calculate() sizes this
        rank's block of servers and solve() exchanges over NVLink inside the library (include/wva_b200.h)."""
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(self.lib.wva_comm_init_rank(self.ctx, world, rank, buf), "wva_comm_init_rank")
        self.world, self.rank = world, rank

    def set_optimizer(self, unlimited: bool, delayed_best_effort: bool = False, saturation_policy="None"):
        """OptimizerSpec of the loaded system, replaced in place (candidates stay valid)."""
        pol = abi.POLICY_NAMES[saturation_policy] if isinstance(saturation_policy, str) else int(saturation_policy)
        self._check(self.lib.wva_set_optimizer(self.ctx, int(bool(unlimited)), int(bool(delayed_best_effort)), pol),
                    "wva_set_optimizer")

    def set_capacity(self, type_count):
        a = np.ascontiguousarray(type_count, np.int32)
        if a.size != self.T:
            raise WvaError(f"set_capacity: {a.size} types, the loaded system has {self.T}")
        self._check(self.lib.wva_set_capacity(self.ctx, a.ctypes.data), "wva_set_capacity")

    # ---- queueing sizing + allocator ------------------------------------------------------
    def load_system(self, sysd: dict):
        st, keep = abi.make_system(sysd)
        self._check(self.lib.wva_load_system(self.ctx, C.byref(st)), "wva_load_system")
        self.S, self.A, self.T = st.n_servers, st.n_acc, st.n_types
        lo, hi = C.c_int32(), C.c_int32()
        self._check(self.lib.wva_comm_shard(self.ctx, C.byref(lo), C.byref(hi)), "wva_comm_shard")
        self.lo, self.hi = lo.value, hi.value

    def calculate(self):
        self._check(self.lib.wva_calculate(self.ctx), "wva_calculate")

    def update_servers(self, arrival, in_tokens, out_tokens, cur_acc, cur_replicas, cur_cost):
        """The per-cycle server columns of the loaded system (ServerLoadSpec, CurrentAlloc), replaced in place; [S]
        arrays.  The servers they change are re-sized or re-valued by the next recalculate()."""
        cols = []
        for (name, dt), a in zip(abi.CYCLE_ARRAYS.items(), (arrival, in_tokens, out_tokens, cur_acc, cur_replicas, cur_cost)):
            a = np.ascontiguousarray(a, dt).reshape(-1)
            if a.size != self.S:
                raise WvaError(f"update_servers: {name} has {a.size} elements, the loaded system has {self.S} servers")
            cols.append(a if a.size else np.zeros(1, dt))
        self._check(self.lib.wva_update_servers(self.ctx, *[a.ctypes.data for a in cols]), "wva_update_servers")

    def recalculate(self):
        """Candidates brought up to date with the update_servers calls since the last calculate / recalculate, equal to a
        calculate().  Returns (servers re-sized, servers re-valued) of this context's block."""
        nr, nv = C.c_int64(), C.c_int64()
        self._check(self.lib.wva_recalculate(self.ctx, C.byref(nr), C.byref(nv)), "wva_recalculate")
        return nr.value, nv.value

    def update_server_set(self, prev, sysd: dict):
        """The loaded system's server set replaced in place by the servers of `sysd` (only its srv_* arrays and n_servers
        are read): prev[i] = index in the loaded system of new server i, or -1 for a new one.  Resident candidates and
        grid follow the new set; the servers that changed are re-sized by the next recalculate() and re-evaluated by the
        next grid_update()."""
        S2 = int(sysd["n_servers"])
        p = np.ascontiguousarray(prev, np.int32).reshape(-1)
        if p.size != S2:
            raise WvaError(f"update_server_set: prev has {p.size} entries, the new set has {S2} servers")
        st, keep = abi.make_system({**sysd, "n_acc": 0, "n_types": 0, "n_models": 0,   # the loaded tables stay
                                    **{k: np.zeros(0, dt) for k, (dt, e) in abi.SYSTEM_ARRAYS.items() if e != "S"}})
        keep.append(p if p.size else np.zeros(1, np.int32))
        self._check(self.lib.wva_update_server_set(self.ctx, S2, keep[-1].ctypes.data, C.byref(st)),
                    "wva_update_server_set")
        self.S = S2
        lo, hi = C.c_int32(), C.c_int32()
        self._check(self.lib.wva_comm_shard(self.ctx, C.byref(lo), C.byref(hi)), "wva_comm_shard")
        self.lo, self.hi = lo.value, hi.value

    def update_tables(self, sysd: dict):
        """The loaded system's accelerator columns (acc_cost, acc_multiplicity, acc_type) and perf_* tables replaced in
        place by those of `sysd` (its n_acc, n_types and n_models must be the loaded ones; its servers, type_count and
        optimizer fields are ignored).  The (server, accelerator) pairs whose perf row or accelerator cost changed are
        re-sized by the next recalculate() and re-evaluated by the next grid_update().  Returns the number of pairs of
        this context's block this call marks for re-sizing."""
        st, keep = abi.make_system({**sysd, "n_servers": 0,   # the loaded servers stay
                                    **{k: np.zeros(0, dt) for k, (dt, e) in abi.SYSTEM_ARRAYS.items() if e == "S"}})
        n = C.c_int64()
        self._check(self.lib.wva_update_tables(self.ctx, C.byref(st), C.byref(n)), "wva_update_tables")
        return n.value

    def solve(self):
        self._check(self.lib.wva_solve(self.ctx), "wva_solve")

    def candidates(self):
        cst, cand = abi.alloc_candidates(self.S, self.A)
        self._check(self.lib.wva_get_candidates(self.ctx, C.byref(cst)), "wva_get_candidates")
        return cand

    def set_candidates(self, cand: dict):
        """Candidates sized elsewhere (another rank's shard, all-gathered) in place of calculate(); [S, A] arrays."""
        for k in abi.CAND_ARRAYS:
            if np.asarray(cand[k]).size != self.S * self.A:
                raise WvaError(f"set_candidates: {k} has {np.asarray(cand[k]).size} elements, the loaded system needs {self.S * self.A}")
        cst, keep = abi.candidates_struct(cand)
        self._check(self.lib.wva_set_candidates(self.ctx, C.byref(cst)), "wva_set_candidates")

    def solution(self):
        sst, sol = abi.alloc_solution(self.S, self.T)
        self._check(self.lib.wva_get_solution(self.ctx, C.byref(sst)), "wva_get_solution")
        return sol

    def optimize(self, sysd: dict):
        """The whole reference path in one call: SetFromSpec -> Calculate -> Optimize -> solution."""
        self.load_system(sysd)
        self.calculate()
        self.solve()
        return self.solution()

    def analyze_grid(self, R: int, full: bool = True, frontier: bool = True):
        S, A = self.hi - self.lo, self.A          # with a communicator: this rank's block of servers
        n = S * A * R
        out = {}
        if full:
            out["ok"] = np.zeros(max(n, 1), dtype=np.uint8)
            for k in ("ttft", "itl", "rho", "tput"):
                out[k] = np.zeros(max(n, 1), dtype=np.float32)
        if frontier:
            out["frontier"] = np.zeros(max(S * A, 1), dtype=np.int32)
        p = lambda k: out[k].ctypes.data if k in out else None
        self._check(self.lib.wva_analyze_grid(self.ctx, R, p("ok"), p("ttft"), p("itl"), p("rho"), p("tput"),
                                              p("frontier")), "wva_analyze_grid")
        self._grid_R = R
        for k in list(out):
            out[k] = out[k][: S * A].reshape(S, A) if k == "frontier" else out[k][:n].reshape(S, A, R)
        return out

    def grid_run(self, R: int, full: bool = False):
        """Grid on the resident system, results stay in HBM (bench: device-resident timing)."""
        self._check(self.lib.wva_grid_run(self.ctx, R, 1 if full else 0), "wva_grid_run")
        self._grid_R = R

    def grid_update(self):
        """The resident grid brought up to date with the update_servers calls since the last grid_run / grid_update,
        equal to a grid_run.  Returns the number of servers of this context's block re-evaluated (load changed)."""
        n = C.c_int64()
        self._check(self.lib.wva_grid_update(self.ctx, C.byref(n)), "wva_grid_update")
        return n.value

    def grid_fetch(self, full: bool = True):
        """The resident grid: frontier [S, A] and, with full (the grid was run with full outputs), ok / ttft / itl / rho /
        tput [S, A, R], as analyze_grid returns them."""
        S, A = self.hi - self.lo, self.A
        R = self._grid_R
        n = S * A * R
        out = {"frontier": np.zeros(max(S * A, 1), dtype=np.int32)}
        if full:
            out["ok"] = np.zeros(max(n, 1), dtype=np.uint8)
            for k in ("ttft", "itl", "rho", "tput"):
                out[k] = np.zeros(max(n, 1), dtype=np.float32)
        p = lambda k: out[k].ctypes.data if k in out else None
        self._check(self.lib.wva_grid_fetch(self.ctx, p("ok"), p("ttft"), p("itl"), p("rho"), p("tput"), p("frontier")),
                    "wva_grid_fetch")
        for k in list(out):
            out[k] = out[k][: S * A].reshape(S, A) if k == "frontier" else out[k][:n].reshape(S, A, R)
        return out

    def grid_fetch_frontier(self):
        S = self.hi - self.lo
        f = np.zeros(max(S * self.A, 1), dtype=np.int32)
        self._check(self.lib.wva_grid_fetch(self.ctx, None, None, None, None, None, f.ctypes.data), "wva_grid_fetch")
        return f[: S * self.A].reshape(S, self.A)

    def mm1k_eval(self, lam, mu, K):
        lam = np.ascontiguousarray(lam, np.float32); mu = np.ascontiguousarray(mu, np.float32)
        K = np.ascontiguousarray(K, np.int32)
        n = lam.size
        names = ("avg_resp", "avg_wait", "avg_serv", "avg_num", "avg_queue", "throughput", "rho")
        out = {"valid": np.zeros(max(n, 1), np.uint8)}
        for k in names:
            out[k] = np.zeros(max(n, 1), np.float32)
        self._check(self.lib.wva_mm1k_eval(self.ctx, n, lam.ctypes.data, mu.ctypes.data, K.ctypes.data,
                                           out["valid"].ctypes.data, *[out[k].ctypes.data for k in names]),
                    "wva_mm1k_eval")
        return {k: v[:n] for k, v in out.items()}

    # ---- saturation + limiter ---------------------------------------------------------------
    def saturation_v1(self, d: dict):
        ist, keep = abi.make_saturation_in(d)
        ost, out = abi.alloc_saturation_out(ist.n_models, ist.n_variants, ist.n_replicas)
        self._check(self.lib.wva_saturation_v1(self.ctx, C.byref(ist), C.byref(ost)), "wva_saturation_v1")
        return out

    def saturation_upload(self, d: dict):
        ist, keep = abi.make_saturation_in(d)
        self._check(self.lib.wva_saturation_upload(self.ctx, C.byref(ist)), "wva_saturation_upload")
        self._sat_dims = (ist.n_models, ist.n_variants, ist.n_replicas)

    def saturation_run(self, detail: bool = False):
        self._check(self.lib.wva_saturation_run(self.ctx, 1 if detail else 0), "wva_saturation_run")

    def saturation_fetch(self, detail: bool = False, fields=None):
        """Results of the last saturation_run.  detail=False: targets, flags and partials only; `fields`: exactly these
        arrays (names of wva_saturation_out) — nothing else is allocated or copied back."""
        M, V, P = self._sat_dims
        ost, out = abi.alloc_saturation_out(M, V, P, only=fields, alloc=self.host_alloc)
        if fields is None and not detail:
            for k in ("var_replica_count", "var_non_saturated", "var_max_kv", "var_max_queue", "var_avg_spare_kv",
                      "var_avg_spare_queue", "rep_saturated", "mod_total_replicas", "mod_non_saturated",
                      "mod_avg_spare_kv", "mod_avg_spare_queue"):
                setattr(ost, k, None)
                out.pop(k, None)
        self._check(self.lib.wva_saturation_fetch(self.ctx, C.byref(ost)), "wva_saturation_fetch")
        return out

    def limit(self, d: dict):
        D = len(d["current"])
        arr = {k: np.ascontiguousarray(d[k], dt) for k, dt in
               (("acc_type", np.int32), ("current", np.int32), ("target", np.int32),
                ("gpus_per_replica", np.int32), ("spare", np.float64), ("cost", np.float64),
                ("type_limit", np.int32))}
        mk = self.host_alloc or (lambda name, n, dt: np.zeros(n, dt))
        out = {"target": mk("limit_target", max(D, 1), np.int32), "gpus_allocated": mk("limit_gpus_allocated", max(D, 1), np.int32),
               "was_limited": mk("limit_was_limited", max(D, 1), np.uint8)}
        self._check(self.lib.wva_limit(self.ctx, D, int(d["n_types"]), arr["acc_type"].ctypes.data,
                                       arr["current"].ctypes.data, arr["target"].ctypes.data,
                                       arr["gpus_per_replica"].ctypes.data, arr["spare"].ctypes.data,
                                       arr["cost"].ctypes.data, arr["type_limit"].ctypes.data,
                                       out["target"].ctypes.data, out["gpus_allocated"].ctypes.data,
                                       out["was_limited"].ctypes.data), "wva_limit")
        return {k: v[:D] for k, v in out.items()}

    # ---- V2 pipeline ------------------------------------------------------------------------------
    def saturation_v2(self, d: dict):
        """SaturationAnalyzer.Analyze arithmetic for a batch of models (see include/wva_b200.h)."""
        ist, ost, keep, out = abi.make_saturation_v2(d)
        self._check(self.lib.wva_saturation_v2(self.ctx, C.byref(ist), C.byref(ost)), "wva_saturation_v2")
        return out

    @staticmethod
    def _batch(d, spec):
        return {k: (None if d.get(k) is None else np.ascontiguousarray(d[k], dt).reshape(-1)) for k, dt in spec}

    def cost_aware_optimize(self, d: dict):
        a = self._batch(d, (("model_variant_off", np.int32), ("mod_required_capacity", np.float64), ("mod_spare_capacity", np.float64),
                            ("mod_has_result", np.uint8), ("var_current", np.int32), ("var_cost", np.float64),
                            ("var_per_replica_capacity", np.float64)))
        M, V = len(a["mod_required_capacity"]), len(a["var_current"])
        tgt = np.zeros(max(V, 1), np.int32)
        p = lambda k: None if a[k] is None or a[k].size == 0 else a[k].ctypes.data
        self._check(self.lib.wva_cost_aware_optimize(self.ctx, M, V, p("model_variant_off"), p("mod_required_capacity"),
                                                     p("mod_spare_capacity"), p("mod_has_result"), p("var_current"), p("var_cost"),
                                                     p("var_per_replica_capacity"), tgt.ctypes.data), "wva_cost_aware_optimize")
        return tgt[:V]

    def enforce(self, d: dict):
        a = self._batch(d, (("model_variant_off", np.int32), ("mod_scale_to_zero_enabled", np.uint8), ("mod_request_count", np.float64),
                            ("mod_request_error", np.uint8), ("var_cost", np.float64), ("var_has_cost", np.uint8)))
        M, V = len(a["mod_request_count"]), len(a["var_cost"])
        tgt = np.ascontiguousarray(d["var_target"], np.int32).reshape(-1).copy()
        if tgt.size == 0:
            tgt = np.zeros(1, np.int32)
        app = np.zeros(max(M, 1), np.uint8)
        p = lambda k: None if a[k] is None or a[k].size == 0 else a[k].ctypes.data
        self._check(self.lib.wva_enforce(self.ctx, M, V, p("model_variant_off"), p("mod_scale_to_zero_enabled"), p("mod_request_count"),
                                         p("mod_request_error"), p("var_cost"), p("var_has_cost"), tgt.ctypes.data, app.ctypes.data),
                    "wva_enforce")
        return tgt[:V], app[:M]

    def pipeline_v2(self, d: dict, var_cost, mod_scale_to_zero_enabled, mod_request_count, mod_request_error=None, var_name_rank=None):
        """analyzer -> cost-aware optimizer -> enforcer chained on the device; returns (analyzer outputs, targets, applied)."""
        ist, ost, keep, out = abi.make_saturation_v2(d)
        V, M = int(d["n_variants"]), int(d["n_models"])
        arr = lambda a, dt: None if a is None else np.ascontiguousarray(a, dt).reshape(-1)
        co, rk = arr(var_cost, np.float64), arr(var_name_rank, np.int32)
        z, rc, re = arr(mod_scale_to_zero_enabled, np.uint8), arr(mod_request_count, np.float64), arr(mod_request_error, np.uint8)
        tgt, app = np.zeros(max(V, 1), np.int32), np.zeros(max(M, 1), np.uint8)
        p = lambda a: None if a is None or a.size == 0 else a.ctypes.data
        self._check(self.lib.wva_pipeline_v2(self.ctx, C.byref(ist), p(co), p(rk), p(z), p(rc), p(re), C.byref(ost), tgt.ctypes.data,
                                             app.ctypes.data), "wva_pipeline_v2")
        return out, tgt[:V], app[:M]

    # ---- observability ------------------------------------------------------------------------
    def timing(self) -> dict:
        t = abi.Timing()
        self._check(self.lib.wva_last_timing(self.ctx, C.byref(t)), "wva_last_timing")
        return {k: getattr(t, k) for k, _ in abi.Timing._fields_}

    def launch_count(self) -> int:
        return int(self.lib.wva_launch_count(self.ctx))

    def microbench_fp64(self):
        a, b = C.c_double(), C.c_double()
        self._check(self.lib.wva_microbench_fp64(self.ctx, C.byref(a), C.byref(b)), "wva_microbench_fp64")
        return a.value, b.value


class K2History:
    """wva_k2_history: the V2 analyzer's k2 priority chain (computeK2) with its rolling history resident on the device
    (include/wva_b200.h).  Registry, all int32: hg_model_off [H+1] / hg_models [G] (history group = modelID -> its model
    groups in visiting order), hg_acc_off [H+1] / hg_acc (its distinct accelerator ids), n_slots store slots.  A registry
    change = export(), a new K2History, import_()."""

    def __init__(self, engine: Engine, hg_model_off, hg_models, hg_acc_off, hg_acc, n_slots: int):
        self.engine, self.lib, self.h = engine, engine.lib, C.c_void_p()
        arr = lambda a: np.ascontiguousarray(a, np.int32).reshape(-1)
        mo, m, ao, a = arr(hg_model_off), arr(hg_models), arr(hg_acc_off), arr(hg_acc)
        p = lambda x: x.ctypes.data if x.size else None
        self.H, self.G, self.n_slots = len(mo) - 1, len(m), int(n_slots)
        engine._check(self.lib.wva_k2_history_create(engine.ctx, self.H, self.G, self.n_slots, p(mo), p(m), p(ao), p(a),
                                                     C.byref(self.h)), "wva_k2_history_create")
        self.K = int(self.lib.wva_k2_history_keys(self.h))

    def close(self):
        if self.h:
            self.lib.wva_k2_history_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def resolve(self, d: dict) -> dict:
        """One cycle (abi.K2_IN columns, optional rep_out_pos + n_out) -> rep_k2, rep_effective, slot_last_rep,
        slot_effective (and out_rep_k2 with rep_out_pos).  Appends to the history once."""
        ist, ost, keep, out = abi.make_k2(d, self.n_slots)
        self.engine._check(self.lib.wva_k2_resolve(self.h, C.byref(ist), C.byref(ost)), "wva_k2_resolve")
        return out

    def export(self) -> dict:
        """every key: hg, acc, bucket, count [K] and values [K, 10] oldest first"""
        K = max(self.K, 1)
        out = {k: np.zeros(K, np.int32) for k in ("hg", "acc", "bucket", "count")}
        out["values"] = np.zeros((K, 10), np.float64)
        self.engine._check(self.lib.wva_k2_history_export(self.h, *(out[k].ctypes.data for k in ("hg", "acc", "bucket", "count", "values"))),
                           "wva_k2_history_export")
        return {k: v[:self.K] for k, v in out.items()}

    def import_(self, e: dict):
        """replace the history with the keys of `e` (export format; keys not listed start empty)"""
        cols = [np.ascontiguousarray(e[k], np.int32).reshape(-1) for k in ("hg", "acc", "bucket", "count")]
        vals = np.ascontiguousarray(e["values"], np.float64).reshape(-1, 10)
        n = len(cols[0])
        if any(len(c) != n for c in cols) or len(vals) != n:
            raise ValueError("import: columns of different lengths")
        p = lambda x: x.ctypes.data if x.size else None
        self.engine._check(self.lib.wva_k2_history_import(self.h, n, *(p(c) for c in cols), p(vals)), "wva_k2_history_import")


class Ingest:
    """wva_ingest: the collector's columnar staging + the streaming reconcile as one CUDA graph (include/wva_b200.h).

    registry: model_variant_off [M+1], variant_slot_off [V+1] (CSR model -> variant -> pod slot; slots of a variant in
    ascending pod-name order).  `cols` / `res` are numpy views of the page-locked arenas the library owns.

    n_types=None: the plain graph (analysis + pre-enforcer targets).  n_types=T >= 0: the decision mode
    (wva_ingest_create_decisions) — the same graph carried on through the enforcer, the decisions and the GPU limiter;
    `dcols` (filled every cycle) and `dres` are then the views of its extra columns and results, and `res` is unchanged."""

    def __init__(self, engine: "Engine", model_variant_off, variant_slot_off, n_types=None):
        self.engine, self.lib = engine, engine.lib
        mvo = np.ascontiguousarray(model_variant_off, np.int32); vso = np.ascontiguousarray(variant_slot_off, np.int32)
        M, V, S = mvo.size - 1, vso.size - 1, int(vso[-1])
        self.M, self.V, self.S = M, V, S
        self.model_variant_off = mvo
        self.T = None if n_types is None else int(n_types)
        self.h = C.c_void_p()
        cst, rst = abi.IngestColumns(), abi.IngestResults()
        if self.T is None:
            engine._check(self.lib.wva_ingest_create(engine.ctx, M, V, S, mvo.ctypes.data, vso.ctypes.data, C.byref(self.h),
                                                     C.byref(cst), C.byref(rst)), "wva_ingest_create")
        else:
            dcst, drst = abi.IngestDecisionColumns(), abi.IngestDecisionResults()
            engine._check(self.lib.wva_ingest_create_decisions(engine.ctx, M, V, S, self.T, mvo.ctypes.data, vso.ctypes.data,
                                                               C.byref(self.h), C.byref(cst), C.byref(rst), C.byref(dcst),
                                                               C.byref(drst)), "wva_ingest_create_decisions")

        def view(p, n, dt):
            if n == 0:
                return np.zeros(0, dt)
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n * np.dtype(dt).itemsize,)).view(dt)

        self.cols = {"kv": view(cst.kv, S, np.float64), "queue": view(cst.queue, S, np.float64), "has": view(cst.has, S, np.uint8),
                     "var_cost": view(cst.var_cost, V, np.float64), "var_current": view(cst.var_current, V, np.int32),
                     "var_desired": view(cst.var_desired, V, np.int32), "var_pending": view(cst.var_pending, V, np.int32),
                     "cfg_kv_threshold": view(cst.cfg_kv_threshold, M, np.float64),
                     "cfg_queue_threshold": view(cst.cfg_queue_threshold, M, np.float64),
                     "cfg_kv_trigger": view(cst.cfg_kv_trigger, M, np.float64),
                     "cfg_queue_trigger": view(cst.cfg_queue_trigger, M, np.float64)}
        self.res = {"var_target": view(rst.var_target, V, np.int32), "var_replica_count": view(rst.var_replica_count, V, np.int32),
                    "var_non_saturated": view(rst.var_non_saturated, V, np.int32),
                    "var_avg_spare_kv": view(rst.var_avg_spare_kv, V, np.float64),
                    "var_avg_spare_queue": view(rst.var_avg_spare_queue, V, np.float64), "mod_flags": view(rst.mod_flags, M, np.uint8),
                    "mod_total_replicas": view(rst.mod_total_replicas, M, np.int32), "partials": view(rst.partials, 4, np.int64)}
        self.dcols = self.dres = None
        if self.T is not None:
            T = self.T
            self.dcols = {"var_accelerator_type": view(dcst.var_accelerator_type, V, np.int32),
                          "var_gpus_per_replica": view(dcst.var_gpus_per_replica, V, np.int32),
                          "mod_scale_to_zero_enabled": view(dcst.mod_scale_to_zero_enabled, M, np.uint8),
                          "mod_request_count": view(dcst.mod_request_count, M, np.float64),
                          "mod_request_error": view(dcst.mod_request_error, M, np.uint8),
                          "type_limit": view(dcst.type_limit, T, np.int32), "enable_limiter": view(dcst.enable_limiter, 1, np.int32)}
            self.dres = {"has_decision": view(drst.has_decision, V, np.uint8), "original_target": view(drst.original_target, V, np.int32),
                         "target": view(drst.target, V, np.int32), "gpus_allocated": view(drst.gpus_allocated, V, np.int32),
                         "was_limited": view(drst.was_limited, V, np.uint8), "action": view(drst.action, V, np.int8),
                         "mod_enforcer_applied": view(drst.mod_enforcer_applied, M, np.uint8)}

    def begin(self):
        self.engine._check(self.lib.wva_ingest_begin(self.h), "wva_ingest_begin")

    def write(self, which: int, slot, value):
        sl = np.ascontiguousarray(slot, np.int32); va = np.ascontiguousarray(value, np.float64)
        self.engine._check(self.lib.wva_ingest_write(self.h, which, sl.size, sl.ctypes.data, va.ctypes.data), "wva_ingest_write")

    def commit(self):
        self.engine._check(self.lib.wva_ingest_commit(self.h), "wva_ingest_commit")
        return self.res

    def close(self):
        if self.h:
            self.lib.wva_ingest_destroy(self.h)
            self.h = None


def _view(p, n, dt):
    """numpy view of n elements of a library-owned page-locked array"""
    if n == 0:
        return np.zeros(0, dt)
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n * np.dtype(dt).itemsize,)).view(dt)


class IngestV2:
    """wva_ingest_v2: the V2 reconcile cycle from metric batch to decisions in two graph launches around the host
    capacity store (include/wva_b200.h).  registry: model_variant_off [M+1], variant_slot_off [V+1] (CSR model ->
    variant -> pod slot, the slots of a variant in ascending pod-name order), var_accelerator [V] (accelerator ids of
    `k2`'s registry), var_store_slot [V] (store slot of namespace|model|variant); `k2` = a K2History whose model groups
    are the models (it must outlive this object).  A cycle: begin(), write() / write_cache_config() and the per-cycle
    columns of `cols`, analyze(), the host step (writes cols["var_fallback_capacity"]), decide(); `res` holds the
    results of the last launch."""

    def __init__(self, engine: "Engine", model_variant_off, variant_slot_off, var_accelerator, var_store_slot, k2: K2History):
        self.engine, self.lib, self.k2 = engine, engine.lib, k2
        mvo = np.ascontiguousarray(model_variant_off, np.int32); vso = np.ascontiguousarray(variant_slot_off, np.int32)
        acc = np.ascontiguousarray(var_accelerator, np.int32); sl = np.ascontiguousarray(var_store_slot, np.int32)
        M, V, S = mvo.size - 1, vso.size - 1, int(vso[-1])
        self.M, self.V, self.S, self.NS = M, V, S, k2.n_slots
        self.model_variant_off, self.variant_slot_off, self.var_accelerator, self.var_store_slot = mvo, vso, acc, sl
        self.h = C.c_void_p()
        cst, rst = abi.IngestV2Columns(), abi.IngestV2Results()
        p = lambda x: x.ctypes.data if x.size else None
        engine._check(self.lib.wva_ingest_v2_create(engine.ctx, M, V, S, mvo.ctypes.data, vso.ctypes.data, p(acc), p(sl), k2.h,
                                                    C.byref(self.h), C.byref(cst), C.byref(rst)), "wva_ingest_v2_create")
        n = {"S": S, "V": V, "M": M, "NS": self.NS, "V1": V + 1}
        self.cols = {k: _view(getattr(cst, k), n[d], dt) for k, dt, d in abi.INGEST_V2_COLUMNS}
        self.res = {k: _view(getattr(rst, k), n[d], dt) for k, dt, d in abi.INGEST_V2_RESULTS}

    def begin(self):
        self.engine._check(self.lib.wva_ingest_v2_begin(self.h), "wva_ingest_v2_begin")

    def write(self, which: int, slot, value):
        sl = np.ascontiguousarray(slot, np.int32); va = np.ascontiguousarray(value, np.float64)
        self.engine._check(self.lib.wva_ingest_v2_write(self.h, which, sl.size, sl.ctypes.data, va.ctypes.data), "wva_ingest_v2_write")

    def write_cache_config(self, slot, num_gpu_blocks, block_size):
        sl = np.ascontiguousarray(slot, np.int32)
        b = np.ascontiguousarray(num_gpu_blocks, np.int64); s = np.ascontiguousarray(block_size, np.int64)
        self.engine._check(self.lib.wva_ingest_v2_write_cache_config(self.h, sl.size, sl.ctypes.data, b.ctypes.data, s.ctypes.data),
                           "wva_ingest_v2_write_cache_config")

    def analyze(self):
        """the first graph launch; analyze_ms = its device time (H2D + pack + k2 chain + D2H, CUDA events)"""
        self.engine._check(self.lib.wva_ingest_v2_analyze(self.h), "wva_ingest_v2_analyze")
        self.analyze_ms = float(self.engine.timing()["saturation_ms"])
        return self.res

    def decide(self):
        """the second graph launch; decide_ms = its device time (H2D + analyzer + optimizer + enforcer + D2H)"""
        self.engine._check(self.lib.wva_ingest_v2_decide(self.h), "wva_ingest_v2_decide")
        self.decide_ms = float(self.engine.timing()["saturation_ms"])
        return self.res

    def close(self):
        if self.h:
            self.lib.wva_ingest_v2_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class Group:
    """wva_group: ONE host process driving several GPUs (what the Go controller does) — n contexts joined by one NCCL
    communicator inside the library, one host thread per device."""

    def __init__(self, devices):
        self.lib = load_library()
        dev = np.ascontiguousarray(devices, np.int32)
        self.g = C.c_void_p()
        rc = self.lib.wva_group_create(dev.ctypes.data, int(dev.size), C.byref(self.g))
        if rc != abi.WVA_OK:
            self.g = None
            raise WvaError(f"wva_group_create({list(dev)}) failed: {self.lib.wva_strerror(rc).decode()}")
        self.n = int(dev.size)

    def close(self):
        if self.g:
            self.lib.wva_group_destroy(self.g)
            self.g = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _err(self, rc, what):
        if rc != abi.WVA_OK:
            details = [self.lib.wva_last_error(self.lib.wva_group_ctx(self.g, i)).decode() for i in range(self.n)]
            raise WvaError(f"{what}: {self.lib.wva_strerror(rc).decode()} {[d for d in details if d]}")

    def optimize(self, sysd: dict):
        """Manager.Optimize over the group (replicated load, sharded sizing, NVLink exchange, allocator)."""
        st, keep = abi.make_system(sysd)
        sst, sol = abi.alloc_solution(st.n_servers, st.n_types)
        self._err(self.lib.wva_group_optimize(self.g, C.byref(st), C.byref(sst)), "wva_group_optimize")
        return sol

    def saturation_v1(self, d: dict):
        ist, keep = abi.make_saturation_in(d)
        ost, out = abi.alloc_saturation_out(ist.n_models, ist.n_variants, ist.n_replicas)
        self._err(self.lib.wva_group_saturation_v1(self.g, C.byref(ist), C.byref(ost)), "wva_group_saturation_v1")
        return out

    def timing(self, i: int) -> dict:
        t = abi.Timing()
        self.lib.wva_last_timing(self.lib.wva_group_ctx(self.g, i), C.byref(t))
        return {k: getattr(t, k) for k, _ in abi.Timing._fields_}
