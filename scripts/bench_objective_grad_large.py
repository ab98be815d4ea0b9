"""Timings of the large-model desirability gradient path on the GPU, qLogEI over a GEOM_MEAN of M bell-shaped targets
with S = 512 base samples, d = 8:
- per-call CUDA-event times (median of 20 calls after 3 warm-up calls) of ``bb_objective_grad`` and
  ``bb_objective_grad_large`` at n = 256, and of ``bb_objective_grad_large`` at n in {320, 512, 1024} and on
  test_gpu_wide.py's d100_n200_m52 model (wide by d), each for M in {2, 8}, at N in {10, 10^4} points and p in {0, 8}
  pending points;
- the bytes of L^-1 (fp32) each call reads, from shapes: both kernels read the lower triangle of every target's L^-1
  in 32 x 32 tiles twice per point, M nb (nb + 1) 4096 bytes with nb = n_pad / 32, and that over the call time;
- the wall time of one 4-D continuous desirability recommend with two targets at n = 1000 (q = 1 and 4), split into
  the raw sweep and final scoring, the device gradient calls and the host L-BFGS-B time, as bench_continuous.py
  splits it.
Prints one JSON line with the card name, power limit and SM clock read in the same run."""
from __future__ import annotations

import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from baybe_b200 import DeviceGP  # noqa: E402
from baybe_b200.continuous import recommend_continuous_hybrid  # noqa: E402
from baybe_b200.synthetic import numeric_grid_workload  # noqa: E402
from scripts.bench_acq_grad_large import linv_bytes_per_point  # noqa: E402
from scripts.bench_continuous import _card  # noqa: E402
from scripts.bench_objective_grad import _events, _gps, _scorer  # noqa: E402


def grad_times(gps, label, ops) -> dict:
    """Per-call times of the ops on the scorer's own arguments (captured from ObjectiveScorer.value_and_grad)."""
    from baybe_b200 import objectives as ob

    out = {}
    M, d = len(gps), gps[0].d
    sc = _scorer(gps)
    for p in (0, 8):
        pend = np.random.default_rng(1).uniform(0, 1, (p, d)) if p else None
        z = sc.base_samples(512, p, 0)
        for N in (10, 10_000):
            x = torch.rand(N, d, device="cuda", generator=torch.Generator("cuda").manual_seed(N))
            seen = {}
            orig = ob.objective_grad_op

            def spy(models, orig=orig, seen=seen):
                op = orig(models)
                return lambda *a: seen.setdefault("args", a) and op(*a)

            ob.objective_grad_op = spy
            try:
                sc.value_and_grad(x, pend, z)
            finally:
                ob.objective_grad_op = orig
            args = seen["args"]
            for name in ops:
                op = getattr(torch.ops.baybe_b200, name)
                ms = _events(lambda: op(*args))
                nbytes = N * sum(linv_bytes_per_point(gp.model.n_pad) for gp in gps)
                out[f"{label}-M{M}-{name}-p{p}-N{N}"] = {"ms": round(ms, 4), "linv_bytes": nbytes,
                                                        "linv_TBps": round(nbytes / (ms * 1e-3) / 1e12, 3)}
    return out


def recommend_times() -> dict:
    res = {}
    sc = _scorer(_gps(2, 1000, 4, seed=2))
    cb = np.array([np.zeros(4), np.ones(4)])
    recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), cb, 1, seed=0)  # warm-up
    for q in (1, 4):
        st: dict = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), cb, q, seed=1, stats=st)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        polish, grad_s = st.get("polish_s", 0.0), st.get("grad_s", 0.0)
        res[f"q{q}"] = {"total": round(total, 3), "raw_sweep_and_final_scoring": round(total - polish, 3),
                        "grad_calls_s": round(grad_s, 3), "lbfgsb_host_s": round(polish - grad_s, 3),
                        "grad_calls": st.get("grad_calls", 0)}
    return res


def main() -> None:
    if not torch.cuda.is_available():
        raise SystemExit("bench_objective_grad_large.py measures on a GPU; none found")
    out = {"card": _card(), "grad": {}, "recommend_n1000_d4_M2_s": {}}
    w = numeric_grid_workload(N=3000, d=100, n=200, seed=11, lengthscale=np.linspace(1.5, 4.0, 100))
    wide = DeviceGP(device="cuda", **w.gp_kwargs())
    for M in (2, 8):
        out["grad"].update(grad_times(_gps(M, 256, 8), "n256", ("objective_grad", "objective_grad_large")))
        for n in (320, 512, 1024):
            out["grad"].update(grad_times(_gps(M, n, 8), f"n{n}", ("objective_grad_large",)))
        out["grad"].update(grad_times([wide] * M, "d100_n200_wide", ("objective_grad_large",)))
    out["recommend_n1000_d4_M2_s"] = recommend_times()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
