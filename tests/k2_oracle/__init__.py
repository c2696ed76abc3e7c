"""ctypes binding of libk2oracle.so (k2_oracle.cpp): the CPU restatement of computeK2 and its rolling history over the
integer registry and inputs of wva_k2_resolve.  Built by __graft_entry__.build() (make -C tests/k2_oracle)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def _load():
    global _lib
    if _lib is None:
        p = os.path.join(_HERE, "libk2oracle.so")
        if not os.path.exists(p):
            raise RuntimeError(f"{p} is missing: run __graft_entry__.build()")
        L = C.CDLL(p)
        L.k2o_create.restype = C.c_void_p
        L.k2o_create.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 4
        L.k2o_destroy.argtypes = [C.c_void_p]
        L.k2o_resolve.argtypes = [C.c_void_p] * 17
        L.k2o_export.argtypes = [C.c_void_p] * 3
        L.k2o_import.argtypes = [C.c_void_p] * 3
        _lib = L
    return _lib


def _a(x, dt):
    a = np.ascontiguousarray(x, dt).reshape(-1)
    return a if a.size else np.zeros(1, dt)


class K2Oracle:
    """Same registry as engine.K2History; resolve(d) takes the same columns (abi.K2_IN) and returns the same outputs
    (without the rep_out_pos scatter); export() -> (count [K], values [K, 10] oldest first) in key order."""

    def __init__(self, hg_model_off, hg_models, hg_acc_off, hg_acc, n_slots):
        self.L = _load()
        self._reg = [_a(hg_model_off, np.int32), _a(hg_models, np.int32), _a(hg_acc_off, np.int32), _a(hg_acc, np.int32)]
        self.H, self.G, self.S = len(np.asarray(hg_model_off)) - 1, len(np.asarray(hg_models)), int(n_slots)
        self.K = 3 * int(np.asarray(hg_acc_off)[-1])
        self.h = self.L.k2o_create(self.H, self.G, self.S, *(r.ctypes.data for r in self._reg))

    def close(self):
        if self.h:
            self.L.k2o_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def resolve(self, d: dict) -> dict | None:
        """-> outputs, or None when the oracle rejects the input (nothing changes then)"""
        P = len(np.asarray(d["rep_total_kv_tokens"]))
        cols = [_a(d["model_replica_off"], np.int32), _a(d["rep_total_kv_tokens"], np.int64), _a(d["rep_tokens_in_use"], np.int64),
                _a(d["rep_queue_length"], np.int64), _a(d["rep_avg_input_tokens"], np.float64),
                _a(d["rep_avg_output_tokens"], np.float64), _a(d["rep_accelerator"], np.int32), _a(d["rep_slot"], np.int32),
                _a(d["cfg_queue_threshold"], np.float64), _a(d["cfg_kv_threshold"], np.float64),
                _a(d["slot_max_batched_tokens"], np.int64), _a(d["slot_max_num_seqs"], np.int64)]
        out = {"rep_k2": np.zeros(max(P, 1), np.int64), "rep_effective": np.zeros(max(P, 1), np.int64),
               "slot_last_rep": np.zeros(max(self.S, 1), np.int32), "slot_effective": np.zeros(max(self.S, 1), np.int64)}
        rc = self.L.k2o_resolve(self.h, *(c.ctypes.data for c in cols), *(o.ctypes.data for o in out.values()))
        if rc:
            return None
        return {"rep_k2": out["rep_k2"][:P], "rep_effective": out["rep_effective"][:P],
                "slot_last_rep": out["slot_last_rep"][:self.S], "slot_effective": out["slot_effective"][:self.S]}

    def export(self):
        count, values = np.zeros(max(self.K, 1), np.int32), np.zeros((max(self.K, 1), 10), np.float64)
        self.L.k2o_export(self.h, count.ctypes.data, values.ctypes.data)
        return count[:self.K], values[:self.K]

    def import_(self, count, values):
        c, v = _a(count, np.int32), np.ascontiguousarray(values, np.float64).reshape(-1, 10)
        if v.size == 0:
            v = np.zeros((1, 10))
        self.L.k2o_import(self.h, c.ctypes.data, v.ctypes.data)
