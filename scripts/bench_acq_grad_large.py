"""Timings of the large-model gradient path on the GPU, qLogEI with S = 512 base samples:
- per-call CUDA-event times (median of 20 calls after 3 warm-up calls) of ``bb_acq_grad`` and ``bb_acq_grad_large``
  at n = 256, d = 8, and of ``bb_acq_grad_large`` at n in {320, 512, 1024} (d = 8) and on test_gpu_wide.py's
  d100_n200_m52 model (wide by d), each at P in {10, 10^4} points and p in {0, 8} pending points;
- the bytes of L^-1 (fp32) each call reads, from shapes: both kernels read the lower triangle in 32 x 32 tiles twice
  per point (v = L^-1 k over row blocks, u = L^-T v over column blocks), nb (nb + 1) 4096 bytes with nb = n_pad / 32,
  and that over the call time;
- the wall time of one 4-D continuous recommend at n = 1000 (q = 1 and 4), split into the raw sweep and final scoring,
  the device gradient calls and the host L-BFGS-B time, as bench_continuous.py splits it.
Prints one JSON line with the card name, power limit and SM clock read in the same run."""
from __future__ import annotations

import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from baybe_b200 import AcqConfig, DeviceGP, sobol_normal_samples, _lib  # noqa: E402
from baybe_b200.continuous import recommend_continuous_hybrid  # noqa: E402
from baybe_b200.synthetic import numeric_grid_workload  # noqa: E402
from scripts.bench_continuous import _card  # noqa: E402
from scripts.bench_objective_grad import _events  # noqa: E402


def _gp(n, d, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (n, d))
    y = np.sin(3 * X).sum(1) + 0.05 * rng.normal(size=n)
    return DeviceGP(device="cuda", train_x=X, train_y=y, bounds=np.array([np.zeros(d), np.ones(d)]),
                    family="matern52", lengthscale=np.full(d, 0.6), noise=1e-3)


def linv_bytes_per_point(n_pad: int) -> int:
    nb = n_pad // 32
    return nb * (nb + 1) * 32 * 32 * 4


def grad_times(gp, label, ops) -> dict:
    out = {}
    d = gp.d
    cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
    for p in (0, 8):
        pend = np.random.default_rng(1).uniform(0, 1, (p, d)) if p else None
        stats = tuple(gp.pending_stats(pend)) if p else (None, None, None, None)
        z = sobol_normal_samples(512, 1 + p, 3).to("cuda", torch.float32).contiguous()
        for P in (10, 10_000):
            x = torch.rand(P, d, device="cuda")
            args = (x, *stats, z, gp.handle, _lib.ACQ_KIND["qLogEI"], cfg.params())
            for name in ops:
                op = getattr(torch.ops.baybe_b200, name)
                ms = _events(lambda: op(*args))
                nbytes = P * linv_bytes_per_point(gp.model.n_pad)
                out[f"{label}-{name}-p{p}-P{P}"] = {"ms": round(ms, 4), "linv_bytes": nbytes,
                                                   "linv_TBps": round(nbytes / (ms * 1e-3) / 1e12, 3)}
    return out


def recommend_times() -> dict:
    res = {}
    gp = _gp(1000, 4, seed=2)
    cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
    cb = np.array([np.zeros(4), np.ones(4)])
    recommend_continuous_hybrid(gp, cfg, np.zeros((1, 0)), cb, 1, seed=0)  # warm-up
    for q in (1, 4):
        st: dict = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        recommend_continuous_hybrid(gp, cfg, np.zeros((1, 0)), cb, q, seed=1, stats=st)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        polish, grad_s = st.get("polish_s", 0.0), st.get("grad_s", 0.0)
        res[f"q{q}"] = {"total": round(total, 3), "raw_sweep_and_final_scoring": round(total - polish, 3),
                        "grad_calls_s": round(grad_s, 3), "lbfgsb_host_s": round(polish - grad_s, 3),
                        "grad_calls": st.get("grad_calls", 0)}
    return res


def main() -> None:
    if not torch.cuda.is_available():
        raise SystemExit("bench_acq_grad_large.py measures on a GPU; none found")
    out = {"card": _card(), "grad": {}, "recommend_n1000_d4_s": {}}
    out["grad"].update(grad_times(_gp(256, 8), "n256", ("acq_grad", "acq_grad_large")))
    for n in (320, 512, 1024):
        out["grad"].update(grad_times(_gp(n, 8), f"n{n}", ("acq_grad_large",)))
    w = numeric_grid_workload(N=3000, d=100, n=200, seed=11, lengthscale=np.linspace(1.5, 4.0, 100))
    out["grad"].update(grad_times(DeviceGP(device="cuda", **w.gp_kwargs()), "d100_n200_wide", ("acq_grad_large",)))
    out["recommend_n1000_d4_s"] = recommend_times()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
