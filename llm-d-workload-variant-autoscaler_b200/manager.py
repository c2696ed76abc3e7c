"""Host-side mirror of the reference's optimizer façade, above the C-ABI.

`Manager(engine, spec).optimize()` is what `pkg/manager.Manager.Optimize` (pkg/manager/manager.go:13-27) followed by
`System.GenerateSolution` (pkg/core/system.go:303-330) is to a reference caller; `spec` is a `config.SystemSpec` in
its JSON shape (pkg/config/types.go:11-215: `acceleratorData.accelerators`, `modelData.models`,
`serviceClassData.serviceClasses`, `serverData.servers`, `optimizerData.optimizer`, `capacityData.count`), so a
fixture written for the reference loads unchanged.  This module is the Python twin of `go/wvab200/wvab200.go`:
names -> ascending-name indices (INTEGRATION.md §3), defaults exactly where the reference applies them, and no
arithmetic of the hot path — that happens behind `wva_calculate` / `wva_solve`.
"""
from __future__ import annotations

import numpy as np

from ._abi import CYCLE_ARRAYS, SYSTEM_ARRAYS

# pkg/config/defaults.go:24-33
DEFAULT_SERVICE_CLASS_NAME = "Free"
DEFAULT_LOW_PRIORITY = 100
DEFAULT_HIGH_PRIORITY = 1
DEFAULT_SERVICE_CLASS_PRIORITY = DEFAULT_LOW_PRIORITY

CUR_ACC_EMPTY = -1     # CurrentAlloc.Accelerator == ""
CUR_ACC_UNKNOWN = -2   # a name that matches no accelerator


def _get(d, *path, default=None):
    for k in path:
        if not isinstance(d, dict) or k not in d:
            return default
        d = d[k]
    return d


class SpecIndex:
    """Name <-> index maps of one flattened spec (ascending names, the order the device path is canonical in)."""

    def __init__(self, acc, types, models, servers):
        self.acc, self.types, self.models, self.servers = acc, types, models, servers
        self.acc_of = {n: i for i, n in enumerate(acc)}
        self.type_of = {n: i for i, n in enumerate(types)}
        self.model_of = {n: i for i, n in enumerate(models)}
        self.server_of = {n: i for i, n in enumerate(servers)}


def flatten_spec(spec: dict):
    """config.SystemSpec (JSON shape) -> (SoA dict for Engine.load_system, SpecIndex).

    Follows System.SetFromSpec (pkg/core/system.go:81-88): maps keyed by name, a repeated name replaces the earlier
    entry; a server whose class or model is unknown keeps its slot (priority default, no target, model -1) because the
    reference keeps such servers and fails them inside Calculate (server.go:55-62, allocation.go:31-47).
    """
    if "system" in spec and "acceleratorData" not in spec:   # config.SystemData wrapper (types.go:6-8)
        spec = spec["system"]
    accs = {a["name"]: a for a in _get(spec, "acceleratorData", "accelerators", default=[]) or []}
    caps = {c["type"]: int(c.get("count", 0)) for c in _get(spec, "capacityData", "count", default=[]) or []}
    perf = _get(spec, "modelData", "models", default=[]) or []
    classes = {c["name"]: c for c in _get(spec, "serviceClassData", "serviceClasses", default=[]) or []}
    servers = {s["name"]: s for s in _get(spec, "serverData", "servers", default=[]) or []}
    opt = _get(spec, "optimizerData", "optimizer", default={}) or {}

    idx = SpecIndex(sorted(accs), sorted({a.get("type", "") for a in accs.values()} | set(caps)),
                    sorted({p["name"] for p in perf}), sorted(servers))
    A, T, M, S = len(idx.acc), len(idx.types), len(idx.models), len(idx.servers)
    d = {
        "n_acc": A, "n_types": T, "n_models": M, "n_servers": S,
        "acc_cost": np.zeros(A, np.float32), "acc_multiplicity": np.zeros(A, np.int32),
        "acc_type": np.zeros(A, np.int32), "type_count": np.zeros(T, np.int32),
    }
    for name, a in accs.items():
        i = idx.acc_of[name]
        d["acc_cost"][i] = np.float32(a.get("cost", 0.0))
        d["acc_multiplicity"][i] = int(a.get("multiplicity", 0))
        d["acc_type"][i] = idx.type_of[a.get("type", "")]
    for t, c in caps.items():
        d["type_count"][idx.type_of[t]] = c                      # a type without a count has capacity 0 (Go map zero value)
    for k, dt in (("perf_alpha", np.float32), ("perf_beta", np.float32), ("perf_gamma", np.float32),
                  ("perf_max_batch", np.int32), ("perf_at_tokens", np.int32), ("perf_acc_count", np.int32),
                  ("perf_present", np.uint8)):
        d[k] = np.zeros((M, A), dt)
    for p in perf:                                               # Model.AddPerfDataFromSpec: (model, acc) replaces
        a = idx.acc_of.get(p.get("acc", ""))
        if a is None:
            continue
        m = idx.model_of[p["name"]]
        sp = p.get("serviceParms", {}) or {}
        d["perf_alpha"][m, a] = np.float32(sp.get("alpha", 0.0))
        d["perf_beta"][m, a] = np.float32(sp.get("beta", 0.0))
        d["perf_gamma"][m, a] = np.float32(sp.get("gamma", 0.0))
        d["perf_max_batch"][m, a] = int(p.get("maxBatchSize", 0))
        d["perf_at_tokens"][m, a] = int(p.get("atTokens", 0))
        d["perf_acc_count"][m, a] = int(p.get("accCount", 0))
        d["perf_present"][m, a] = 1
    prio, targets = {}, {}
    for name, c in classes.items():                              # NewServiceClass clamps (serviceclass.go:28-31)
        p = int(c.get("priority", 0))
        if p < DEFAULT_HIGH_PRIORITY or p > DEFAULT_LOW_PRIORITY:
            p = DEFAULT_SERVICE_CLASS_PRIORITY
        prio[name] = p
        targets[name] = {t["model"]: t for t in c.get("modelTargets", []) or []}
    for k, dt in (("srv_model", np.int32), ("srv_priority", np.int32), ("srv_min_replicas", np.int32),
                  ("srv_max_batch", np.int32), ("srv_keep_acc", np.uint8), ("srv_target_present", np.uint8),
                  ("srv_slo_ttft", np.float32), ("srv_slo_itl", np.float32), ("srv_slo_tps", np.float32),
                  ("srv_arrival", np.float32), ("srv_in_tokens", np.int32), ("srv_out_tokens", np.int32),
                  ("srv_cur_acc", np.int32), ("srv_cur_replicas", np.int32), ("srv_cur_cost", np.float32)):
        d[k] = np.zeros(S, dt)
    for name, s in servers.items():
        i = idx.server_of[name]
        cls = s.get("class", "") or DEFAULT_SERVICE_CLASS_NAME   # server.go:38-41
        d["srv_model"][i] = idx.model_of.get(s.get("model", ""), -1)
        d["srv_priority"][i] = prio.get(cls, DEFAULT_SERVICE_CLASS_PRIORITY)     # server.go:92-97
        t = targets.get(cls, {}).get(s.get("model", ""))
        if t is not None:
            d["srv_target_present"][i] = 1
            d["srv_slo_ttft"][i] = np.float32(t.get("slo-ttft", 0.0))
            d["srv_slo_itl"][i] = np.float32(t.get("slo-itl", 0.0))
            d["srv_slo_tps"][i] = np.float32(t.get("slo-tps", 0.0))
        d["srv_min_replicas"][i] = int(s.get("minNumReplicas", 0))
        d["srv_max_batch"][i] = int(s.get("maxBatchSize", 0))
        d["srv_keep_acc"][i] = 1 if s.get("keepAccelerator", False) else 0
        cur = s.get("currentAlloc", {}) or {}
        load = cur.get("load", {}) or {}
        d["srv_arrival"][i] = np.float32(load.get("arrivalRate", 0.0))
        d["srv_in_tokens"][i] = int(load.get("avgInTokens", 0))
        d["srv_out_tokens"][i] = int(load.get("avgOutTokens", 0))
        ca = cur.get("accelerator", "") or ""
        d["srv_cur_acc"][i] = CUR_ACC_EMPTY if ca == "" else idx.acc_of.get(ca, CUR_ACC_UNKNOWN)
        d["srv_cur_replicas"][i] = int(cur.get("numReplicas", 0))
        d["srv_cur_cost"][i] = np.float32(cur.get("cost", 0.0))
    d["unlimited"] = bool(opt.get("unlimited", False))
    d["delayed_best_effort"] = bool(opt.get("delayedBestEffort", False))
    d["saturation_policy"] = opt.get("saturationPolicy", "None")   # unknown strings -> default (config.go:28-41)
    return d, idx


def _equal_except(old: dict, new: dict, free) -> bool:
    """True when two flattened specs have the same keys and every array and scalar not named in `free` is equal (arrays
    byte for byte, with the same dtype and shape)."""
    if old.keys() != new.keys():
        return False
    for k, a in old.items():
        if k in free:
            continue
        b = new[k]
        if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
            a, b = np.asarray(a), np.asarray(b)
            if a.dtype != b.dtype or a.shape != b.shape or a.tobytes() != b.tobytes():
                return False
        elif a != b:
            return False
    return True


def differs_only_in_cycle_columns(old: dict, new: dict) -> bool:
    """True when two flattened specs describe the same system up to the per-cycle server columns (loads and current
    allocations, CYCLE_ARRAYS): every other array equal byte for byte, every scalar equal."""
    return _equal_except(old, new, CYCLE_ARRAYS)


# the accelerator columns and the perf tables: what Engine.update_tables replaces in place
TABLE_ARRAYS = tuple(k for k, (dt, e) in SYSTEM_ARRAYS.items() if e in ("A", "MA"))


def differs_only_in_tables(old: dict, new: dict) -> bool:
    """True when two flattened specs describe systems of the same shape (accelerators, types, models, servers) that
    differ only in the accelerator columns and perf tables (TABLE_ARRAYS: costs, multiplicities, types, perf data) and
    the per-cycle server columns: Engine.update_tables (+ update_servers) brings the device from one to the other."""
    for k in TABLE_ARRAYS:
        if k not in old or k not in new:
            return False
        a, b = np.asarray(old[k]), np.asarray(new[k])
        if a.dtype != b.dtype or a.shape != b.shape:
            return False
    return _equal_except(old, new, set(TABLE_ARRAYS) | set(CYCLE_ARRAYS))


def server_set_prev(old_index: SpecIndex, old: dict, new_index: SpecIndex, new: dict):
    """The `prev` map of Engine.update_server_set from the system on the device (old) to a new one, or None when the
    two flattened specs differ in more than their servers: prev[i] = old index of new server i (by name), -1 for a new
    server.  Every array and scalar that is not a server column (accelerators, types and capacity, models and perf
    data, the optimizer) must be equal byte for byte; the server set and every srv_* column may change."""
    if old.keys() != new.keys():
        return None
    for k, a in old.items():
        if k.startswith("srv_") or k == "n_servers":
            continue
        b = new[k]
        if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
            a, b = np.asarray(a), np.asarray(b)
            if a.dtype != b.dtype or a.shape != b.shape or a.tobytes() != b.tobytes():
                return None
        elif a != b:
            return None
    return np.array([old_index.server_of.get(name, -1) for name in new_index.servers], np.int32)


def solution_to_spec(sol: dict, idx: SpecIndex, spec_servers: dict | None = None) -> dict:
    """Solution arrays -> config.AllocationSolution JSON shape (System.GenerateSolution, system.go:303-330):
    a server with no allocation is absent; the zero-load allocation has accelerator ""."""
    out = {}
    for i, name in enumerate(idx.servers):
        st = int(sol["state"][i])
        if st == 0:
            continue
        load = ((spec_servers or {}).get(name, {}).get("currentAlloc", {}) or {}).get("load", {})
        out[name] = {
            "accelerator": idx.acc[int(sol["acc"][i])] if st == 1 else "",
            "numReplicas": int(sol["num_replicas"][i]), "maxBatch": int(sol["batch_size"][i]),
            "cost": float(sol["cost"][i]), "itlAverage": float(sol["itl"][i]), "ttftAverage": float(sol["ttft"][i]),
            "load": dict(load),
        }
    return {"allocations": out}


class Manager:
    """`manager.NewManager(system, optimizer)` + `Optimize()` for one SystemSpec, on the device."""

    def __init__(self, engine, spec: dict):
        self.engine = engine
        self.spec = spec["system"] if "system" in spec and "acceleratorData" not in spec else spec
        self.sysd, self.index = flatten_spec(self.spec)
        self._sized = False        # the engine holds self.sysd and its candidates from calculate / recalculate

    def optimize(self) -> dict:
        """Returns the AllocationSolution (JSON shape).  Raises WvaError where the reference returns an error."""
        self._sized = False
        sol = self.engine.optimize(self.sysd)
        self._sized = True
        return self._solution(sol)

    def update(self, spec: dict) -> dict:
        """One reconcile cycle on a rebuilt SystemSpec, the same result as `Manager(engine, spec).optimize()`.  When the
        new spec differs from the one on the device only in server loads and current allocations, those columns are
        replaced in place and only the servers they changed are re-sized or re-valued (update_servers -> recalculate
        -> solve).  When accelerator columns or perf data changed too, with the same shapes, the tables are replaced in
        place first and only the (server, accelerator) pairs that read a changed row are re-sized (update_tables ->
        update_servers -> recalculate -> solve).  Any other change reloads the system (load_system -> calculate ->
        solve)."""
        spec = spec["system"] if "system" in spec and "acceleratorData" not in spec else spec
        sysd, index = flatten_spec(spec)
        incremental = self._sized and differs_only_in_cycle_columns(self.sysd, sysd)
        tables = self._sized and not incremental and differs_only_in_tables(self.sysd, sysd)
        self.spec, self.sysd, self.index, self._cand = spec, sysd, index, None
        self._sized = False
        eng = self.engine
        if incremental or tables:
            if tables:
                eng.update_tables(sysd)
            eng.update_servers(*(sysd[k] for k in CYCLE_ARRAYS))
            eng.recalculate()
        else:
            eng.load_system(sysd)
            eng.calculate()
        self._sized = True
        eng.solve()
        return self._solution(eng.solution())

    def _solution(self, sol: dict) -> dict:
        self.last_solution = sol
        servers = {s["name"]: s for s in _get(self.spec, "serverData", "servers", default=[]) or []}
        return solution_to_spec(sol, self.index, servers)

    def analyze_model(self, server_name: str) -> dict:
        """interfaces.ModelAnalyzer.AnalyzeModel as internal/modelanalyzer implements it (analyzer.go:24-33, utils.go:9-25):
        Server.Calculate for one variant server -> {"Allocations": {accelerator: ModelAcceleratorAllocation}}; an unknown
        server gives the empty response.  The device sizes every server of the spec in the same launch; the required-QPS
        fields are the adapter's float32 product MaxArrvRatePerReplica * 1000, widened."""
        i = self.index.server_of.get(server_name)
        if i is None:
            return {"Allocations": {}}
        if getattr(self, "_cand", None) is None:
            self._sized = False
            self.engine.load_system(self.sysd)
            self.engine.calculate()
            self._sized = True
            self._cand = self.engine.candidates()
        c = self._cand
        out = {}
        for a, acc in enumerate(self.index.acc):
            st = int(c["state"][i, a])
            if st == 0:
                continue                                         # nil allocation: not in Server.AllAllocations()
            qps = float(np.float32(c["max_arrv_rate"][i, a]) * np.float32(1000.0))
            out[acc] = {"Allocation": {"accelerator": acc if st == 1 else "", "numReplicas": int(c["num_replicas"][i, a]),
                                       "maxBatch": int(c["batch_size"][i, a]), "cost": float(c["cost"][i, a]),
                                       "value": float(c["value"][i, a]), "itlAverage": float(c["itl"][i, a]),
                                       "ttftAverage": float(c["ttft"][i, a]), "rho": float(c["rho"][i, a]),
                                       "maxArrvRatePerReplica": float(c["max_arrv_rate"][i, a])},
                        "RequiredPrefillQPS": qps, "RequiredDecodeQPS": qps, "Reason": "markovian analysis"}
        return {"Allocations": out}

    def allocation_by_type(self) -> dict:
        """System.AllocateByType (system.go:271-300): accelerator type -> (count, limit, cost) of the last solution."""
        sol = self.last_solution
        used = (np.asarray(sol["state"]) == 1) & (self.sysd["srv_model"] >= 0)   # acc == nil || model == nil -> skipped
        used_types = set(int(t) for t in self.sysd["acc_type"][np.asarray(sol["acc"])[used]])
        return {name: {"count": int(sol["type_count"][t]), "limit": int(self.sysd["type_count"][t]),
                       "cost": float(sol["type_cost"][t])}
                for t, name in enumerate(self.index.types) if t in used_types}
