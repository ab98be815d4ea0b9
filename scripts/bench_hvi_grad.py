"""Timings of the Pareto gradient path on the GPU: ``bb_hvi_grad`` per call at n = 256, d = 20, S = 512, 10 points (the
default n_restarts), M in {2, 3, 4} targets, qEHVI and qLogEHVI, 0 and 8 pending points (CUDA events, median of 50
calls after 5 warm-up calls; the pending decompositions are built once, as in a greedy step), and wall times of one
continuous recommend (baybe_b200/continuous.py, 4 continuous parameters) at q = 1 and q = 4, split into the raw sweep
and final scoring, the host box decompositions, and L-BFGS-B (device gradient calls and host time).  Prints one JSON
line with the card name, power limit and SM clock read in the same run."""
from __future__ import annotations

import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from baybe_b200 import AcqConfig, DeviceGP  # noqa: E402
from baybe_b200 import multiobjective as mo  # noqa: E402
from baybe_b200.continuous import recommend_continuous_hybrid  # noqa: E402
from scripts.bench_continuous import _card  # noqa: E402
from scripts.bench_objective_grad import _events  # noqa: E402


def _scorer(kind, M, n, d, seed=0):
    gps = []
    for m in range(M):
        rng = np.random.default_rng(seed + m)
        X = rng.uniform(0, 1, (n, d))
        y = np.sin(3 * X[:, :4]).sum(1) * (1 if m % 2 == 0 else -1) + 0.3 * m + 0.05 * rng.normal(size=n)
        gps.append(DeviceGP(device="cuda", train_x=X, train_y=y, bounds=np.array([np.zeros(d), np.ones(d)]),
                            family="matern52", lengthscale=np.full(d, 0.6), noise=1e-3))
    a = np.array([1.0, -1.0, 1.0, -1.0][:M])
    b = np.zeros(M)
    X0 = torch.from_numpy(np.random.default_rng(seed + 99).uniform(0, 1, (24, d))).float().cuda()
    front = np.stack([gp.posterior(X0)[0].double().cpu().numpy() for gp in gps], 1) * a + b
    return mo.HviScorer(gps, AcqConfig(kind=kind), a, b, mo.compute_ref_point(front), front)


def main():
    out = {"card": _card(), "hvi_grad_ms": {}, "recommend_s": {}}
    n, d, S, N = 256, 20, 512, 10
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.uniform(0, 1, (N, d))).float()
    for M in (2, 3, 4):
        for kind in ("qEHVI", "qLogEHVI"):
            sc = _scorer(kind, M, n, d)
            for P in (0, 8):
                pend = rng.uniform(0, 1, (P, d)) if P else None
                z = sc.base_samples(S, P, 3)
                sc.value_and_grad(x, pend, z)  # builds the step's decompositions once
                out["hvi_grad_ms"][f"M{M}-{kind}-P{P}"] = round(_events(lambda: sc.value_and_grad(x, pend, z),
                                                                        reps=50, warm=5), 4)
    for q in (1, 4):
        sc = _scorer("qLogEHVI", 2, n, 4, seed=5)
        real = mo.box_decomposition
        box = {"s": 0.0}

        def timed(*a, **k):
            t0 = time.perf_counter()
            r = real(*a, **k)
            box["s"] += time.perf_counter() - t0
            return r

        mo.box_decomposition = timed
        try:
            stats = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), np.array([np.zeros(4), np.ones(4)]), q,
                                        n_samples=S, seed=7, n_raw_samples=64, n_restarts=10, stats=stats)
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
        finally:
            mo.box_decomposition = real
        polish = stats.get("polish_s", 0.0)
        out["recommend_s"][f"q{q}"] = {"total": round(total, 3), "box_decompositions": round(box["s"], 3),
                                        "lbfgsb": round(polish, 3), "grad_calls_s": round(stats.get("grad_s", 0.0), 3),
                                        "grad_calls": stats.get("grad_calls", 0),
                                        "raw_and_final_scoring": round(total - polish - box["s"], 3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
