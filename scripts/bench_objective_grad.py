"""Timings of the desirability gradient path on the GPU: ``bb_objective_grad`` per call at N in {10, 1e4}, M in {2, 4,
8} targets, n = 256, S = 512, d = 8, P in {0, 8} (CUDA events, median of 20 calls after 3 warm-up calls; the
pending-point conditioning is built once, as in a greedy step), and wall times of a desirability recommend (baybe_b200/continuous.py): a 4-D continuous space (q = 1, 8) and the config-3 hybrid shape
(1296 configurations x 4 continuous parameters, q = 16), split into raw sweeps and final scoring, device gradient calls
and host L-BFGS-B time.  Prints one JSON line with the card name, power limit and SM clock read in the same run."""
from __future__ import annotations

import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from baybe_b200 import AcqConfig, DeviceGP  # noqa: E402
from baybe_b200.continuous import recommend_continuous_hybrid  # noqa: E402
from baybe_b200.objectives import CompiledObjective, ObjectiveScorer  # noqa: E402
from scripts.bench_continuous import _card  # noqa: E402


def _gps(M, n, d, seed=0):
    out = []
    for m in range(M):
        rng = np.random.default_rng(seed + m)
        X = rng.uniform(0, 1, (n, d))
        y = np.sin(3 * X).sum(1) + 0.3 * m + 0.05 * rng.normal(size=n)
        out.append(DeviceGP(device="cuda", train_x=X, train_y=y, bounds=np.array([np.zeros(d), np.ones(d)]),
                            family="matern52", lengthscale=np.full(d, 0.6), noise=1e-3))
    return out


def _scorer(gps):
    M = len(gps)
    progs = [[("BELL", (1.0 + 0.1 * m, 0.8, 0.0))] for m in range(M)]
    comp = CompiledObjective([f"t{m}" for m in range(M)], progs, "GEOM_MEAN", np.full(M, 1.0 / M))
    return ObjectiveScorer(gps, AcqConfig("qLogEI", best_f=0.5), comp)


def _events(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        t.append(a.elapsed_time(b))
    return float(np.median(t))


def main():
    out = {"card": _card(), "objective_grad_ms": {}, "recommend_s": {}}
    d, n, S = 8, 256, 512
    for M in (2, 4, 8):
        sc = _scorer(_gps(M, n, d))
        for P in (0, 8):
            pend = np.random.default_rng(1).uniform(0, 1, (P, d)) if P else None
            z = sc.base_samples(S, P, 0)
            for N in (10, 10_000):
                x = torch.from_numpy(np.random.default_rng(2).uniform(0, 1, (N, d))).float()
                xd = x.cuda()
                out["objective_grad_ms"][f"M{M}_P{P}_N{N}"] = _events(lambda: sc.value_and_grad(xd, pend, z))
    # wall time of a desirability recommend, split as DESIGN.md section 4.3 does
    for name, (nc, dc, q) in {"cont4_q1": (1, 4, 1), "cont4_q8": (1, 4, 8), "config3_q16": (1296, 4, 16)}.items():
        dd = 4 if nc > 1 else 0
        gps = _gps(2, 64, dd + dc, seed=5)
        sc = _scorer(gps)
        disc = (np.random.default_rng(3).uniform(0, 1, (nc, dd)) if nc > 1 else np.zeros((1, 0)))
        cb = np.array([np.zeros(dc), np.ones(dc)])
        stats = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        recommend_continuous_hybrid(sc, sc.cfg, disc, cb, q, seed=1, stats=stats)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        out["recommend_s"][name] = {"total": total, "device_grad_calls": stats.get("grad_s", 0.0),
                                    "grad_calls": stats.get("grad_calls", 0),
                                    "lbfgsb_host": stats.get("polish_s", 0.0) - stats.get("grad_s", 0.0),
                                    "raw_sweeps_and_scoring": total - stats.get("polish_s", 0.0)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
