"""Timings of the gradient path on the GPU: ``bb_acq_grad`` per call at P in {10, 1e4, 1e5}, n in {64, 256},
p in {0, 8} (CUDA events, 20 calls after 3 warm-up calls), and wall times of the continuous / hybrid optimiser
(baybe_b200/continuous.py): a 4-D continuous space (q = 1, 8) and the config-3 hybrid shape (1296 configurations x 4
continuous parameters, qLogEI, q = 16), split into raw sweep, device gradient calls and host L-BFGS-B time.  Prints
one JSON line with the card name and power limit read in the same run."""
from __future__ import annotations

import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from baybe_b200 import AcqConfig, DeviceGP, sobol_normal_samples  # noqa: E402
from baybe_b200.continuous import recommend_continuous_hybrid  # noqa: E402


def _gp(n, d, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (n, d))
    y = np.sin(3 * X).sum(1) + 0.05 * rng.normal(size=n)
    return DeviceGP(device="cuda", train_x=X, train_y=y, bounds=np.array([np.zeros(d), np.ones(d)]),
                    family="matern52", lengthscale=np.full(d, 0.6), noise=1e-3)


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, pl, clk = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def grad_times() -> list[dict]:
    out = []
    d = 8
    for n in (64, 256):
        gp = _gp(n, d)
        cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
        for p in (0, 8):
            pend = np.random.default_rng(1).uniform(0, 1, (p, d)) if p else None
            z = sobol_normal_samples(512, 1 + p, 3)
            for P in (10, 10_000, 100_000):
                x = torch.rand(P, d, device="cuda")
                for _ in range(3):
                    gp.value_and_grad(cfg, x, z, pend)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(20):
                    gp.value_and_grad(cfg, x, z, pend)
                e1.record()
                torch.cuda.synchronize()
                out.append({"n": n, "p": p, "P": P, "ms_per_call": e0.elapsed_time(e1) / 20})
    return out


def optimiser_times() -> dict:
    res = {}
    gp = _gp(64, 4, seed=2)
    cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
    cb = np.array([np.zeros(4), np.ones(4)])
    for q in (1, 8):
        recommend_continuous_hybrid(gp, cfg, np.zeros((1, 0)), cb, 1, seed=0)  # warm-up
        torch.cuda.synchronize()
        st: dict = {}
        t0 = time.perf_counter()
        recommend_continuous_hybrid(gp, cfg, np.zeros((1, 0)), cb, q, seed=1, stats=st)
        torch.cuda.synchronize()
        res[f"continuous_4d_q{q}_s"] = time.perf_counter() - t0
        res[f"continuous_4d_q{q}_grad_calls"] = st.get("grad_calls", 0)
    lv = np.linspace(0, 1, 6)
    disc = np.array(np.meshgrid(lv, lv, lv, lv, indexing="ij")).reshape(4, -1).T
    rng = np.random.default_rng(3)
    X = np.hstack([disc[rng.integers(0, len(disc), 256)], rng.uniform(0, 1, (256, 4))])
    y = np.sin(3 * X).sum(1)
    gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=np.array([np.zeros(8), np.ones(8)]), family="matern52",
                  lengthscale=np.full(8, 0.6), noise=1e-3)
    cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
    st = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    recommend_continuous_hybrid(gp, cfg, disc, cb, 16, seed=1, stats=st)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    res.update({"config3_q16_s": total, "config3_grad_calls_s": st.get("grad_s", 0.0),
                "config3_lbfgsb_host_s": st.get("polish_s", 0.0) - st.get("grad_s", 0.0),
                "config3_raw_sweep_and_rest_s": total - st.get("polish_s", 0.0),
                "config3_grad_calls": st.get("grad_calls", 0)})
    return res


def main() -> None:
    if not torch.cuda.is_available():
        raise SystemExit("bench_continuous.py measures on a GPU; none found")
    info = _card()
    print(json.dumps({**info, "acq_grad": grad_times(), **optimiser_times()}))


if __name__ == "__main__":
    main()
