"""Seeded synthetic inputs for the BASELINE.json configs (SURVEY.md §8(d)).

One counter-based RNG (numpy Philox), seed 0xB2005EED, stream id = config
number; generated once on the host and fed unchanged to the oracle and to the
GPU path.  Nothing here computes any part of the hot path.
"""
from __future__ import annotations

import numpy as np

SEED = 0xB2005EED

# (TTFT ms, ITL ms, TPS) per service class and class priorities (SURVEY.md §8d)
CLASS_SLOS = [(500.0, 24.0, 0.0), (2000.0, 80.0, 0.0), (0.0, 200.0, 0.0)]
CLASS_PRIORITIES = [1, 5, 10]


def _rng(stream: int):
    return np.random.Generator(np.random.Philox(key=SEED + (int(stream) << 32)))


def queue_system(S: int, A: int, N: int, n_classes: int = 3, stream: int = 2, unlimited: bool = True,
                 R: int | None = None, zero_load_frac: float = 0.05, infeasible_frac: float = 0.02,
                 saturation_policy="None", delayed_best_effort: bool = False):
    """Queueing-path system: S servers (one model each), A accelerator variants, max batch N.

    R (replica levels) only scales the arrival-rate range; defaults to N as SURVEY §8d pins N = R.
    """
    R = N if R is None else R
    g = _rng(stream)
    T = min(A, 8)
    a = np.arange(A)
    d = {
        "n_acc": A, "n_types": T, "n_models": S, "n_servers": S,
        "acc_cost": (25.0 * 1.35 ** a).astype(np.float32),
        "acc_multiplicity": np.array([1, 2, 4, 8], dtype=np.int32)[a % 4],
        "acc_type": (a % T).astype(np.int32),
        "type_count": np.full(T, 2**31 - 1, dtype=np.int32),
    }
    speed = (0.8 ** a)[None, :]
    d["perf_alpha"] = (g.uniform(4.0, 20.0, (S, A)) * speed).astype(np.float32)
    d["perf_beta"] = (g.uniform(0.01, 0.3, (S, A)) * speed).astype(np.float32)
    d["perf_gamma"] = (g.uniform(5e-4, 2e-2, (S, A)) * speed).astype(np.float32)
    in_tok = np.clip(np.floor(g.lognormal(np.log(512.0), 0.8, S)), 16, 8192).astype(np.int32)
    out_tok = np.clip(np.floor(g.lognormal(np.log(160.0), 0.7, S)), 8, 2048).astype(np.int32)
    d["perf_max_batch"] = np.full((S, A), N, dtype=np.int32)
    d["perf_at_tokens"] = np.repeat(out_tok[:, None], A, axis=1).astype(np.int32)  # derived N stays N
    d["perf_acc_count"] = g.integers(1, 3, (S, A)).astype(np.int32)
    d["perf_present"] = np.ones((S, A), dtype=np.uint8)
    arrival = 60.0 * np.exp(g.uniform(np.log(0.05), np.log(2.0 * R), S))
    arrival[g.random(S) < zero_load_frac] = 0.0
    cls = (np.arange(S) % n_classes).astype(np.int64)
    scale = g.uniform(0.8, 1.25, S)
    slo = np.array(CLASS_SLOS[:n_classes], dtype=np.float64)[cls] * scale[:, None]
    bad = g.random(S) < infeasible_frac
    slo[bad, 1] = 0.01  # unsatisfiable ITL -> bisection ind < 0 -> infeasible
    d.update({
        "srv_model": np.arange(S, dtype=np.int32),
        "srv_priority": np.array(CLASS_PRIORITIES[:n_classes], dtype=np.int32)[cls],
        "srv_min_replicas": np.ones(S, dtype=np.int32),
        "srv_max_batch": np.zeros(S, dtype=np.int32),
        "srv_keep_acc": np.zeros(S, dtype=np.uint8),
        "srv_target_present": np.ones(S, dtype=np.uint8),
        "srv_slo_ttft": slo[:, 0].astype(np.float32),
        "srv_slo_itl": slo[:, 1].astype(np.float32),
        "srv_slo_tps": slo[:, 2].astype(np.float32),
        "srv_arrival": arrival.astype(np.float32),
        "srv_in_tokens": in_tok, "srv_out_tokens": out_tok,
        "srv_cur_acc": np.full(S, -1, dtype=np.int32),
        "srv_cur_replicas": np.zeros(S, dtype=np.int32),
        "srv_cur_cost": np.zeros(S, dtype=np.float32),
        "unlimited": unlimited, "delayed_best_effort": delayed_best_effort,
        "saturation_policy": saturation_policy,
    })
    return d


def baseline_config(cfg: int, scale: float = 1.0):
    """BASELINE.json configs 1-3 (queueing path).  scale < 1 shrinks S for CPU-side tests."""
    if cfg == 1:
        return queue_system(max(1, int(10 * scale)), 4, 32, n_classes=1, stream=1)
    if cfg == 2:
        return queue_system(max(1, int(1000 * scale)), 16, 128, n_classes=3, stream=2)
    if cfg == 3:
        return queue_system(max(1, int(100000 * scale)), 32, 256, n_classes=3, stream=3, unlimited=False)
    raise ValueError(cfg)


def limit_capacity(sysd: dict, unconstrained_type_count, fraction: float = 0.6):
    """Set per-type capacity to `fraction` of the unconstrained demand so the cap binds (SURVEY §8d)."""
    out = dict(sysd)
    out["type_count"] = np.maximum(1, np.floor(np.asarray(unconstrained_type_count, dtype=np.float64) * fraction)
                                   ).astype(np.int32)
    out["unlimited"] = False
    return out


def shard_system(sysd: dict, rank: int, world: int):
    """Model-sharded partition (SURVEY §8e): servers s with s % world == rank, tables replicated.

    The shard keeps the perf rows of the models its servers run, once per model, and renumbers them.  A server with an
    unknown model (srv_model < 0) keeps -1: it has no candidates, as in the whole system (Server.Calculate).
    """
    S, A = int(sysd["n_servers"]), int(sysd["n_acc"])
    idx = np.arange(rank, S, world)
    out = dict(sysd)
    for k, v in sysd.items():
        if k.startswith("srv_"):
            out[k] = np.asarray(v)[idx]
    smod = np.asarray(sysd["srv_model"])[idx]
    known = smod >= 0
    models, local = np.unique(smod[known], return_inverse=True)
    for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_max_batch", "perf_at_tokens", "perf_acc_count",
              "perf_present"):
        out[k] = np.ascontiguousarray(np.asarray(sysd[k]).reshape(int(sysd["n_models"]), A)[models])
    sm = np.full(len(idx), -1, dtype=np.int32)
    sm[known] = local
    out["srv_model"] = sm
    out["n_models"] = len(models)
    out["n_servers"] = len(idx)
    return out, idx


def saturation_batch(M: int, V_per_model: int = 32, stream: int = 4, max_replicas: int = 8,
                     transition_frac: float = 0.03):
    """BASELINE config 4: V1 saturation inputs (SURVEY §8d cfg 4)."""
    g = _rng(stream)
    V = M * V_per_model
    nrep = g.integers(1, max_replicas + 1, V).astype(np.int32)
    off = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(nrep, out=off[1:])
    P = int(off[-1])
    assert P < 2**31
    # per-model load level so that every branch occurs: idle models (scale-down safe), busy models
    # (no action) and hot models (scale-up)
    level = np.repeat(np.repeat(g.choice([0, 1, 2], M, p=[0.35, 0.35, 0.30]), V_per_model), nrep)
    kv = g.beta(2.0, 3.0, P)
    kv[level == 0] *= 0.45                                                # idle: spare KV ~0.6
    hot_m = level == 2                                                    # hot: spare KV ~0.06 < trigger 0.1
    kv[hot_m] = g.uniform(0.68, 0.795, int(hot_m.sum()))
    hot = g.random(P) < 0.10
    kv[hot] = g.uniform(0.8, 1.0, int(hot.sum()))
    queue = g.poisson(1.5, P).astype(np.int64)
    burst = g.random(P) < 0.05
    queue[burst] += g.poisson(8.0, int(burst.sum()))
    a = np.arange(V) % V_per_model
    cost = (25.0 * 1.35 ** (a % 16)) * (1.0 + (a // 16))  # distinct per variant within a model
    current = nrep.copy()
    desired = np.zeros(V, dtype=np.int32)
    pending = (g.random(V) < 0.05).astype(np.int32)
    trans_models = np.flatnonzero(g.random(M) < transition_frac)
    tv = trans_models * V_per_model + g.integers(0, V_per_model, len(trans_models))
    desired[tv] = current[tv] + 1
    return {
        "n_models": M, "n_variants": V, "n_replicas": P,
        "model_variant_off": (np.arange(M + 1, dtype=np.int64) * V_per_model).astype(np.int32),
        "variant_replica_off": off.astype(np.int32),
        "rep_kv": kv.astype(np.float64), "rep_queue": queue,
        "var_cost": cost.astype(np.float64), "var_current": current, "var_desired": desired,
        "var_pending": pending,
        "cfg_kv_threshold": np.full(M, 0.8), "cfg_queue_threshold": np.full(M, 5.0),
        "cfg_kv_trigger": np.full(M, 0.1), "cfg_queue_trigger": np.full(M, 3.0),
    }


def limiter_batch(D: int, T: int = 8, stream: int = 6, tightness: float = 0.6):
    """Decisions for the GPU-count limiter (pipeline.DefaultLimiter.Limit)."""
    g = _rng(stream)
    acc_type = g.integers(0, T, D).astype(np.int32)
    acc_type[g.random(D) < 0.01] = -1  # AcceleratorName == ""
    current = g.integers(0, 9, D).astype(np.int32)
    delta = g.integers(-1, 4, D).astype(np.int32)
    target = np.maximum(current + delta, 0).astype(np.int32)
    gpr = np.array([0, 1, 1, 2, 4, 8], dtype=np.int32)[g.integers(0, 6, D)]
    spare = np.round(g.random(D), 2)  # 2 decimals -> plenty of exact ties on SpareCapacity
    cost = (25.0 * 1.35 ** g.integers(0, 8, D)).astype(np.float64)
    used = np.zeros(T, dtype=np.int64)
    req = np.zeros(T, dtype=np.int64)
    for t in range(T):
        m = acc_type == t
        used[t] = int((current[m].astype(np.int64) * gpr[m]).sum())
        up = m & (target > current)
        req[t] = int(((target[up] - current[up]).astype(np.int64) * np.maximum(gpr[up], 1)).sum())
    limit = (used + np.floor(req * tightness)).astype(np.int32)
    return {"acc_type": acc_type, "current": current, "target": target, "gpus_per_replica": gpr,
            "spare": spare.astype(np.float64), "cost": cost, "type_limit": limit, "n_types": T}
