"""ctypes image of include/wva_b200.h (the C-ABI of the H100 hot path).

Only struct layouts, constants and numpy<->pointer helpers live here; nothing in
this module computes anything.  Both the product wrapper (``engine.py``) and the
test-side oracle wrapper (``tests/oracle_lib.py``) marshal through these structs
so that the two sides are fed byte-identical buffers.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

WVA_OK = 0
WVA_ERR_ARG, WVA_ERR_CUDA, WVA_ERR_NO_DEVICE, WVA_ERR_STATE, WVA_ERR_NOMEM, WVA_ERR_LIMIT = 1, 2, 3, 4, 5, 6
POLICY_NONE, POLICY_PRIORITY_EXHAUSTIVE, POLICY_PRIORITY_ROUND_ROBIN, POLICY_ROUND_ROBIN = 0, 1, 2, 3
POLICY_NAMES = {
    "None": POLICY_NONE,
    "PriorityExhaustive": POLICY_PRIORITY_EXHAUSTIVE,
    "PriorityRoundRobin": POLICY_PRIORITY_ROUND_ROBIN,
    "RoundRobin": POLICY_ROUND_ROBIN,
}
ALLOC_NONE, ALLOC_ACC, ALLOC_EMPTY = 0, 1, 2
CUR_ACC_EMPTY, CUR_ACC_UNKNOWN = -1, -2
SAT_SCALE_UP, SAT_SCALE_DOWN_SAFE, SAT_IN_TRANSITION, SAT_KV_TRIGGERED, SAT_QUEUE_TRIGGERED = 1, 2, 4, 8, 16

_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)
_u8p = C.POINTER(C.c_uint8)

_CT = {np.dtype(np.float32): _f32p, np.dtype(np.float64): _f64p, np.dtype(np.int32): _i32p,
       np.dtype(np.int64): _i64p, np.dtype(np.uint8): _u8p}


def ptr(a):
    """numpy array -> typed ctypes pointer (None -> NULL of unknown type is not allowed here)."""
    assert a.flags["C_CONTIGUOUS"], "C-ABI buffers must be contiguous"
    return a.ctypes.data_as(_CT[a.dtype])


class System(C.Structure):
    _fields_ = [
        ("n_acc", C.c_int32), ("n_types", C.c_int32),
        ("acc_cost", _f32p), ("acc_multiplicity", _i32p), ("acc_type", _i32p), ("type_count", _i32p),
        ("n_models", C.c_int32),
        ("perf_alpha", _f32p), ("perf_beta", _f32p), ("perf_gamma", _f32p),
        ("perf_max_batch", _i32p), ("perf_at_tokens", _i32p), ("perf_acc_count", _i32p), ("perf_present", _u8p),
        ("n_servers", C.c_int32),
        ("srv_model", _i32p), ("srv_priority", _i32p), ("srv_min_replicas", _i32p), ("srv_max_batch", _i32p),
        ("srv_keep_acc", _u8p), ("srv_target_present", _u8p),
        ("srv_slo_ttft", _f32p), ("srv_slo_itl", _f32p), ("srv_slo_tps", _f32p),
        ("srv_arrival", _f32p), ("srv_in_tokens", _i32p), ("srv_out_tokens", _i32p),
        ("srv_cur_acc", _i32p), ("srv_cur_replicas", _i32p), ("srv_cur_cost", _f32p),
        ("unlimited", C.c_uint8), ("delayed_best_effort", C.c_uint8), ("saturation_policy", C.c_int32),
    ]


class Candidates(C.Structure):
    _fields_ = [("state", _u8p), ("num_replicas", _i32p), ("batch_size", _i32p), ("cost", _f32p),
                ("value", _f32p), ("itl", _f32p), ("ttft", _f32p), ("rho", _f32p), ("max_arrv_rate", _f32p),
                ("n_solves", _i32p)]


class Solution(C.Structure):
    _fields_ = [("state", _u8p), ("acc", _i32p), ("num_replicas", _i32p), ("batch_size", _i32p),
                ("cost", _f32p), ("value", _f32p), ("itl", _f32p), ("ttft", _f32p), ("rho", _f32p),
                ("max_arrv_rate", _f32p), ("type_count", _i64p), ("type_cost", _f64p)]


class Timing(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("calculate_ms", C.c_float), ("solve_ms", C.c_float),
                ("grid_ms", C.c_float), ("saturation_ms", C.c_float), ("limit_ms", C.c_float),
                ("d2h_ms", C.c_float), ("chain_solves", C.c_int64), ("chain_states", C.c_int64),
                ("overflow_pairs", C.c_int64), ("exchange_ms", C.c_float), ("sizer_kernel", C.c_int32),
                ("greedy_heap_pushes", C.c_int64), ("greedy_events", C.c_int64), ("certify_fallbacks", C.c_int64)]


class SaturationIn(C.Structure):
    _fields_ = [("n_models", C.c_int64), ("n_variants", C.c_int64), ("n_replicas", C.c_int64),
                ("model_variant_off", _i32p), ("variant_replica_off", _i32p),
                ("rep_kv", _f64p), ("rep_queue", _i64p),
                ("var_cost", _f64p), ("var_current", _i32p), ("var_desired", _i32p), ("var_pending", _i32p),
                ("var_has_state", _u8p),
                ("cfg_kv_threshold", _f64p), ("cfg_queue_threshold", _f64p),
                ("cfg_kv_trigger", _f64p), ("cfg_queue_trigger", _f64p)]


class SaturationOut(C.Structure):
    _fields_ = [("var_target", _i32p), ("var_replica_count", _i32p), ("var_non_saturated", _i32p),
                ("var_max_kv", _f64p), ("var_max_queue", _i64p), ("var_avg_spare_kv", _f64p),
                ("var_avg_spare_queue", _f64p), ("rep_saturated", _u8p),
                ("mod_total_replicas", _i32p), ("mod_non_saturated", _i32p), ("mod_avg_spare_kv", _f64p),
                ("mod_avg_spare_queue", _f64p), ("mod_flags", _u8p), ("partials", _i64p),
                ("partials_all", _i64p)]


# ---- field specs used to build/validate the SoA dicts ------------------------------------
SYSTEM_ARRAYS = {
    # name: (dtype, size-expression over (A, T, M, S))
    "acc_cost": (np.float32, "A"), "acc_multiplicity": (np.int32, "A"), "acc_type": (np.int32, "A"),
    "type_count": (np.int32, "T"),
    "perf_alpha": (np.float32, "MA"), "perf_beta": (np.float32, "MA"), "perf_gamma": (np.float32, "MA"),
    "perf_max_batch": (np.int32, "MA"), "perf_at_tokens": (np.int32, "MA"), "perf_acc_count": (np.int32, "MA"),
    "perf_present": (np.uint8, "MA"),
    "srv_model": (np.int32, "S"), "srv_priority": (np.int32, "S"), "srv_min_replicas": (np.int32, "S"),
    "srv_max_batch": (np.int32, "S"), "srv_keep_acc": (np.uint8, "S"), "srv_target_present": (np.uint8, "S"),
    "srv_slo_ttft": (np.float32, "S"), "srv_slo_itl": (np.float32, "S"), "srv_slo_tps": (np.float32, "S"),
    "srv_arrival": (np.float32, "S"), "srv_in_tokens": (np.int32, "S"), "srv_out_tokens": (np.int32, "S"),
    "srv_cur_acc": (np.int32, "S"), "srv_cur_replicas": (np.int32, "S"), "srv_cur_cost": (np.float32, "S"),
}

# the per-cycle server columns wva_update_servers replaces, in its argument order
CYCLE_ARRAYS = {"srv_arrival": np.float32, "srv_in_tokens": np.int32, "srv_out_tokens": np.int32,
                "srv_cur_acc": np.int32, "srv_cur_replicas": np.int32, "srv_cur_cost": np.float32}

CAND_ARRAYS = {"state": np.uint8, "num_replicas": np.int32, "batch_size": np.int32, "cost": np.float32,
               "value": np.float32, "itl": np.float32, "ttft": np.float32, "rho": np.float32,
               "max_arrv_rate": np.float32, "n_solves": np.int32}

SOL_ARRAYS = {"state": np.uint8, "acc": np.int32, "num_replicas": np.int32, "batch_size": np.int32,
              "cost": np.float32, "value": np.float32, "itl": np.float32, "ttft": np.float32,
              "rho": np.float32, "max_arrv_rate": np.float32}


def _size(expr, A, T, M, S):
    return {"A": A, "T": T, "MA": M * A, "S": S}[expr]


def make_system(sysd: dict):
    """dict of numpy arrays + scalars -> (System struct, keepalive list).

    ``sysd`` keys: every name in SYSTEM_ARRAYS plus n_acc, n_types, n_models,
    n_servers, unlimited, delayed_best_effort, saturation_policy.
    """
    A, T, M, S = int(sysd["n_acc"]), int(sysd["n_types"]), int(sysd["n_models"]), int(sysd["n_servers"])
    st = System()
    keep = []
    st.n_acc, st.n_types, st.n_models, st.n_servers = A, T, M, S
    for name, (dt, expr) in SYSTEM_ARRAYS.items():
        a = np.ascontiguousarray(sysd[name], dtype=dt).reshape(-1)
        n = _size(expr, A, T, M, S)
        if a.size != n:
            raise ValueError(f"{name}: expected {n} elements, got {a.size}")
        if a.size == 0:  # keep a valid non-NULL pointer for empty arrays
            a = np.zeros(1, dtype=dt)
        keep.append(a)
        setattr(st, name, ptr(a))
    st.unlimited = 1 if sysd.get("unlimited", True) else 0
    st.delayed_best_effort = 1 if sysd.get("delayed_best_effort", False) else 0
    pol = sysd.get("saturation_policy", POLICY_NONE)
    st.saturation_policy = POLICY_NAMES.get(pol, POLICY_NONE) if isinstance(pol, str) else int(pol)
    return st, keep


def alloc_candidates(S: int, A: int):
    arrs = {k: np.zeros(max(S * A, 1), dtype=dt) for k, dt in CAND_ARRAYS.items()}
    st = Candidates()
    for k, a in arrs.items():
        setattr(st, k, ptr(a))
    return st, {k: a[: S * A].reshape(S, A) if S * A else a[:0].reshape(S, A) for k, a in arrs.items()}


def candidates_struct(cand: dict):
    """dict of [S,A] arrays (as returned by alloc_candidates) -> Candidates struct + keepalive."""
    st = Candidates()
    keep = []
    for k, dt in CAND_ARRAYS.items():
        a = np.ascontiguousarray(cand[k], dtype=dt).reshape(-1)
        if a.size == 0:
            a = np.zeros(1, dtype=dt)
        keep.append(a)
        setattr(st, k, ptr(a))
    return st, keep


def alloc_solution(S: int, T: int):
    arrs = {k: np.zeros(max(S, 1), dtype=dt) for k, dt in SOL_ARRAYS.items()}
    arrs["type_count"] = np.zeros(max(T, 1), dtype=np.int64)
    arrs["type_cost"] = np.zeros(max(T, 1), dtype=np.float64)
    st = Solution()
    for k, a in arrs.items():
        setattr(st, k, ptr(a))
    out = {k: a[:S] for k, a in arrs.items() if k in SOL_ARRAYS}
    out["type_count"] = arrs["type_count"][:T]
    out["type_cost"] = arrs["type_cost"][:T]
    return st, out


def make_saturation_in(d: dict):
    st = SaturationIn()
    keep = []
    M = int(d["n_models"]); V = int(d["n_variants"]); P = int(d["n_replicas"])
    st.n_models, st.n_variants, st.n_replicas = M, V, P
    spec = {"model_variant_off": (np.int32, M + 1), "variant_replica_off": (np.int32, V + 1),
            "rep_kv": (np.float64, P), "rep_queue": (np.int64, P),
            "var_cost": (np.float64, V), "var_current": (np.int32, V), "var_desired": (np.int32, V),
            "var_pending": (np.int32, V),
            "cfg_kv_threshold": (np.float64, M), "cfg_queue_threshold": (np.float64, M),
            "cfg_kv_trigger": (np.float64, M), "cfg_queue_trigger": (np.float64, M)}
    for name, (dt, n) in spec.items():
        a = np.ascontiguousarray(d[name], dtype=dt).reshape(-1)
        if a.size != n:
            raise ValueError(f"{name}: expected {n} elements, got {a.size}")
        if a.size == 0:
            a = np.zeros(1, dtype=dt)
        keep.append(a)
        setattr(st, name, ptr(a))
    hs = d.get("var_has_state")
    if hs is not None:
        a = np.ascontiguousarray(hs, dtype=np.uint8).reshape(-1)
        if a.size != V:
            raise ValueError("var_has_state size")
        if a.size == 0:
            a = np.zeros(1, dtype=np.uint8)
        keep.append(a)
        st.var_has_state = ptr(a)
    return st, keep


def alloc_saturation_out(M: int, V: int, P: int, only=None, alloc=None):
    spec = {"var_target": (np.int32, V), "var_replica_count": (np.int32, V), "var_non_saturated": (np.int32, V),
            "var_max_kv": (np.float64, V), "var_max_queue": (np.int64, V), "var_avg_spare_kv": (np.float64, V),
            "var_avg_spare_queue": (np.float64, V), "rep_saturated": (np.uint8, P),
            "mod_total_replicas": (np.int32, M), "mod_non_saturated": (np.int32, M),
            "mod_avg_spare_kv": (np.float64, M), "mod_avg_spare_queue": (np.float64, M),
            "mod_flags": (np.uint8, M), "partials": (np.int64, 4), "partials_all": (np.int64, 4)}
    st = SaturationOut()
    out = {}
    for name, (dt, n) in spec.items():
        if only is not None and name not in only:
            setattr(st, name, None)
            continue
        a = alloc(name, max(n, 1), dt) if alloc else np.zeros(max(n, 1), dtype=dt)
        setattr(st, name, ptr(a))
        out[name] = a[:n]
    return st, out


# ---- V2 pipeline ---------------------------------------------------------------------------------------------------
_i64p = C.POINTER(C.c_int64)


class SaturationV2In(C.Structure):
    _fields_ = [("n_models", C.c_int64), ("n_variants", C.c_int64), ("n_replicas", C.c_int64),
                ("model_variant_off", _i32p), ("variant_replica_off", _i32p),
                ("rep_total_kv_tokens", _i64p), ("rep_tokens_in_use", _i64p), ("rep_queue_length", _i64p),
                ("rep_avg_input_tokens", _f64p), ("rep_avg_output_tokens", _f64p), ("rep_prefix_hit_rate", _f64p),
                ("rep_k2", _i64p), ("rep_slice_order", _i32p),
                ("var_current", _i32p), ("var_pending", _i32p), ("var_fallback_capacity", _f64p),
                ("cfg_kv_threshold", _f64p), ("cfg_scale_up_threshold", _f64p), ("cfg_scale_down_boundary", _f64p),
                ("sched_queue_size", _i64p), ("sched_queue_bytes", _i64p)]


class SaturationV2Out(C.Structure):
    _fields_ = [("rep_k1", _i64p), ("rep_effective", _i64p), ("rep_demand", _i64p), ("rep_saturated", _u8p),
                ("var_ready", _i32p), ("var_per_replica_capacity", _f64p), ("var_total_capacity", _f64p),
                ("var_total_demand", _f64p), ("var_utilization", _f64p),
                ("mod_total_supply", _f64p), ("mod_total_demand", _f64p), ("mod_utilization", _f64p),
                ("mod_required_capacity", _f64p), ("mod_spare_capacity", _f64p)]


SAT_V2_IN = {"model_variant_off": (np.int32, "M1"), "variant_replica_off": (np.int32, "V1"),
             "rep_total_kv_tokens": (np.int64, "P"), "rep_tokens_in_use": (np.int64, "P"), "rep_queue_length": (np.int64, "P"),
             "rep_avg_input_tokens": (np.float64, "P"), "rep_avg_output_tokens": (np.float64, "P"),
             "rep_prefix_hit_rate": (np.float64, "P"), "rep_k2": (np.int64, "P"), "rep_slice_order": (np.int32, "P"),
             "var_current": (np.int32, "V"), "var_pending": (np.int32, "V"), "var_fallback_capacity": (np.float64, "V"),
             "cfg_kv_threshold": (np.float64, "M"), "cfg_scale_up_threshold": (np.float64, "M"),
             "cfg_scale_down_boundary": (np.float64, "M"), "sched_queue_size": (np.int64, "M"), "sched_queue_bytes": (np.int64, "M")}
SAT_V2_OPTIONAL = ("rep_slice_order", "sched_queue_size", "sched_queue_bytes")
SAT_V2_OUT = {"rep_k1": (np.int64, "P"), "rep_effective": (np.int64, "P"), "rep_demand": (np.int64, "P"),
              "rep_saturated": (np.uint8, "P"), "var_ready": (np.int32, "V"), "var_per_replica_capacity": (np.float64, "V"),
              "var_total_capacity": (np.float64, "V"), "var_total_demand": (np.float64, "V"), "var_utilization": (np.float64, "V"),
              "mod_total_supply": (np.float64, "M"), "mod_total_demand": (np.float64, "M"), "mod_utilization": (np.float64, "M"),
              "mod_required_capacity": (np.float64, "M"), "mod_spare_capacity": (np.float64, "M")}


def make_saturation_v2(d: dict):
    M, V, P = int(d["n_models"]), int(d["n_variants"]), int(d["n_replicas"])
    n = {"M": M, "V": V, "P": P, "M1": M + 1, "V1": V + 1}
    ist, ost, keep, out = SaturationV2In(), SaturationV2Out(), [], {}
    ist.n_models, ist.n_variants, ist.n_replicas = M, V, P
    for name, (dt, dim) in SAT_V2_IN.items():
        if name in SAT_V2_OPTIONAL and d.get(name) is None:
            setattr(ist, name, None)
            continue
        a = np.ascontiguousarray(d[name], dtype=dt).reshape(-1)
        if a.size != n[dim]:
            raise ValueError(f"{name}: expected {n[dim]} elements, got {a.size}")
        if a.size == 0:
            a = np.zeros(1, dt)
        keep.append(a)
        setattr(ist, name, ptr(a))
    for name, (dt, dim) in SAT_V2_OUT.items():
        a = np.zeros(max(n[dim], 1), dtype=dt)
        setattr(ost, name, ptr(a))
        out[name] = a[:n[dim]]
    return ist, ost, keep, out


# ---- k2 priority chain with its rolling history ----------------------------------------------------------------------
class K2In(C.Structure):
    _fields_ = [("n_model_groups", C.c_int64), ("n_replicas", C.c_int64), ("model_replica_off", _i32p),
                ("rep_total_kv_tokens", _i64p), ("rep_tokens_in_use", _i64p), ("rep_queue_length", _i64p),
                ("rep_avg_input_tokens", _f64p), ("rep_avg_output_tokens", _f64p), ("rep_accelerator", _i32p),
                ("rep_slot", _i32p), ("rep_out_pos", _i32p), ("n_out", C.c_int64),
                ("slot_max_batched_tokens", _i64p), ("slot_max_num_seqs", _i64p),
                ("cfg_queue_threshold", _f64p), ("cfg_kv_threshold", _f64p)]


class K2Out(C.Structure):
    _fields_ = [("rep_k2", _i64p), ("rep_effective", _i64p), ("out_rep_k2", _i64p), ("slot_last_rep", _i32p),
                ("slot_effective", _i64p)]


# name -> (dtype, extent): G model groups, P replicas, S store slots
K2_IN = {"model_replica_off": (np.int32, "G1"), "rep_total_kv_tokens": (np.int64, "P"), "rep_tokens_in_use": (np.int64, "P"),
         "rep_queue_length": (np.int64, "P"), "rep_avg_input_tokens": (np.float64, "P"),
         "rep_avg_output_tokens": (np.float64, "P"), "rep_accelerator": (np.int32, "P"), "rep_slot": (np.int32, "P"),
         "rep_out_pos": (np.int32, "P"), "slot_max_batched_tokens": (np.int64, "S"), "slot_max_num_seqs": (np.int64, "S"),
         "cfg_queue_threshold": (np.float64, "G"), "cfg_kv_threshold": (np.float64, "G")}
K2_OUT = {"rep_k2": (np.int64, "P"), "rep_effective": (np.int64, "P"), "out_rep_k2": (np.int64, "N"),
          "slot_last_rep": (np.int32, "S"), "slot_effective": (np.int64, "S")}


def make_k2(d: dict, n_slots: int):
    """d: the K2_IN columns (rep_out_pos may be absent or None; then n_out is ignored) -> (in, out, keep-alive, outputs)."""
    G, P = len(d["model_replica_off"]) - 1, len(d["rep_total_kv_tokens"])
    has_pos = d.get("rep_out_pos") is not None
    N = int(d.get("n_out", 0)) if has_pos else 0
    n = {"G": G, "G1": G + 1, "P": P, "S": n_slots, "N": N}
    ist, ost, keep, out = K2In(), K2Out(), [], {}
    ist.n_model_groups, ist.n_replicas, ist.n_out = G, P, N
    for name, (dt, dim) in K2_IN.items():
        if name == "rep_out_pos" and not has_pos:
            setattr(ist, name, None)
            continue
        a = np.ascontiguousarray(d[name], dtype=dt).reshape(-1)
        if a.size != n[dim]:
            raise ValueError(f"{name}: expected {n[dim]} elements, got {a.size}")
        if a.size == 0:
            a = np.zeros(1, dt)
        keep.append(a)
        setattr(ist, name, ptr(a))
    for name, (dt, dim) in K2_OUT.items():
        if name == "out_rep_k2" and not has_pos:
            setattr(ost, name, None)
            continue
        a = np.zeros(max(n[dim], 1), dtype=dt)
        setattr(ost, name, ptr(a))
        out[name] = a[:n[dim]]
    return ist, ost, keep, out


# ---- ingest ------------------------------------------------------------------------------------------------------------
class IngestColumns(C.Structure):
    _fields_ = [("n_slots", C.c_int64), ("n_variants", C.c_int64), ("n_models", C.c_int64),
                ("kv", _f64p), ("queue", _f64p), ("has", _u8p), ("var_cost", _f64p), ("var_current", _i32p),
                ("var_desired", _i32p), ("var_pending", _i32p), ("cfg_kv_threshold", _f64p),
                ("cfg_queue_threshold", _f64p), ("cfg_kv_trigger", _f64p), ("cfg_queue_trigger", _f64p)]


class IngestResults(C.Structure):
    _fields_ = [("var_target", _i32p), ("var_replica_count", _i32p), ("var_non_saturated", _i32p),
                ("var_avg_spare_kv", _f64p), ("var_avg_spare_queue", _f64p), ("mod_flags", _u8p),
                ("mod_total_replicas", _i32p), ("partials", _i64p)]


class IngestDecisionColumns(C.Structure):
    _fields_ = [("n_types", C.c_int32), ("var_accelerator_type", _i32p), ("var_gpus_per_replica", _i32p),
                ("mod_scale_to_zero_enabled", _u8p), ("mod_request_count", _f64p), ("mod_request_error", _u8p),
                ("type_limit", _i32p), ("enable_limiter", _i32p)]


class IngestDecisionResults(C.Structure):
    _fields_ = [("has_decision", _u8p), ("original_target", _i32p), ("target", _i32p), ("gpus_allocated", _i32p),
                ("was_limited", _u8p), ("action", C.POINTER(C.c_int8)), ("mod_enforcer_applied", _u8p)]


VEC_KV_CACHE_USAGE, VEC_QUEUE_LENGTH = 0, 1


# ---- V2 ingest ---------------------------------------------------------------------------------------------------------
class IngestV2Columns(C.Structure):
    _fields_ = [("n_slots", C.c_int64), ("n_variants", C.c_int64), ("n_models", C.c_int64), ("n_store_slots", C.c_int64),
                ("kv", _f64p), ("queue", _f64p), ("num_gpu_blocks", _i64p), ("block_size", _i64p),
                ("avg_output_tokens", _f64p), ("avg_input_tokens", _f64p), ("prefix_hit_rate", _f64p), ("has", _u8p),
                ("var_cost", _f64p), ("var_current", _i32p), ("var_pending", _i32p), ("var_name_rank", _i32p),
                ("cfg_kv_threshold", _f64p), ("cfg_queue_threshold", _f64p), ("cfg_scale_up_threshold", _f64p),
                ("cfg_scale_down_boundary", _f64p), ("mod_scale_to_zero_enabled", _u8p), ("mod_request_count", _f64p),
                ("mod_request_error", _u8p), ("slot_max_batched_tokens", _i64p), ("slot_max_num_seqs", _i64p),
                ("var_fallback_capacity", _f64p)]


class IngestV2Results(C.Structure):
    _fields_ = [("variant_replica_off", _i32p), ("rep_pod", _i32p), ("rep_total_kv_tokens", _i64p), ("slot_last_rep", _i32p),
                ("slot_effective", _i64p), ("var_no_data", _u8p), ("mod_has_request", _u8p),
                ("mod_avg_input_tokens", _f64p), ("mod_avg_output_tokens", _f64p),
                ("var_optimizer_target", _i32p), ("var_target", _i32p), ("var_action", C.POINTER(C.c_int8)),
                ("mod_enforced", _u8p), ("var_ready", _i32p), ("var_per_replica_capacity", _f64p),
                ("var_total_capacity", _f64p), ("var_total_demand", _f64p), ("var_utilization", _f64p),
                ("mod_total_supply", _f64p), ("mod_total_demand", _f64p), ("mod_utilization", _f64p),
                ("mod_required_capacity", _f64p), ("mod_spare_capacity", _f64p)]


VEC_AVG_OUTPUT_TOKENS, VEC_AVG_INPUT_TOKENS, VEC_PREFIX_CACHE_HIT_RATE = 2, 3, 4
CACHE_LABEL_ABSENT = -(1 << 63)          # a cache_config_info label that is absent or does not parse

# (name, dtype, dimension) of the V2 ingest arenas: S pod slots, V variants, M models, NS store slots
INGEST_V2_COLUMNS = [("kv", np.float64, "S"), ("queue", np.float64, "S"), ("num_gpu_blocks", np.int64, "S"),
                     ("block_size", np.int64, "S"), ("avg_output_tokens", np.float64, "S"),
                     ("avg_input_tokens", np.float64, "S"), ("prefix_hit_rate", np.float64, "S"), ("has", np.uint8, "S"),
                     ("var_cost", np.float64, "V"), ("var_current", np.int32, "V"), ("var_pending", np.int32, "V"),
                     ("var_name_rank", np.int32, "V"), ("cfg_kv_threshold", np.float64, "M"),
                     ("cfg_queue_threshold", np.float64, "M"), ("cfg_scale_up_threshold", np.float64, "M"),
                     ("cfg_scale_down_boundary", np.float64, "M"), ("mod_scale_to_zero_enabled", np.uint8, "M"),
                     ("mod_request_count", np.float64, "M"), ("mod_request_error", np.uint8, "M"),
                     ("slot_max_batched_tokens", np.int64, "NS"), ("slot_max_num_seqs", np.int64, "NS"),
                     ("var_fallback_capacity", np.float64, "V")]
INGEST_V2_RESULTS = [("variant_replica_off", np.int32, "V1"), ("rep_pod", np.int32, "S"), ("rep_total_kv_tokens", np.int64, "S"),
                     ("slot_last_rep", np.int32, "NS"), ("slot_effective", np.int64, "NS"), ("var_no_data", np.uint8, "V"),
                     ("mod_has_request", np.uint8, "M"), ("mod_avg_input_tokens", np.float64, "M"),
                     ("mod_avg_output_tokens", np.float64, "M"), ("var_optimizer_target", np.int32, "V"),
                     ("var_target", np.int32, "V"), ("var_action", np.int8, "V"), ("mod_enforced", np.uint8, "M"),
                     ("var_ready", np.int32, "V"), ("var_per_replica_capacity", np.float64, "V"),
                     ("var_total_capacity", np.float64, "V"), ("var_total_demand", np.float64, "V"),
                     ("var_utilization", np.float64, "V"), ("mod_total_supply", np.float64, "M"),
                     ("mod_total_demand", np.float64, "M"), ("mod_utilization", np.float64, "M"),
                     ("mod_required_capacity", np.float64, "M"), ("mod_spare_capacity", np.float64, "M")]
