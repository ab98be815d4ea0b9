"""Timings of qNIPV's gradient path on the GPU (csrc/nipvgrad.cu): ``bb_nipv_phi`` per image and ``bb_nipv_grad`` per
evaluation at n = 256, d = 20, P = 10, M in {4096, 65536, 1e6}, |C| in {0, 8} (CUDA events, 20 calls after 3 warm-up
calls), the bandwidth ``bb_nipv_grad`` achieves against the bytes it must stream ((r + d) M 4 B per 16-point tile,
over the H100 SXM's 3.35 TB/s), and wall times of a whole continuous recommend (4-D, 4096 integration points, n = 64,
q = 1 and q = 4) split into conditioning (with the image), L-BFGS-B polish and raw sweep plus final scoring.  Prints
one JSON line with the card name and power limit read in the same run."""
from __future__ import annotations

import json
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from baybe_b200 import AcqConfig, DeviceGP  # noqa: E402
from baybe_b200 import nipv as nv  # noqa: E402
from baybe_b200.continuous import recommend_continuous_hybrid  # noqa: E402
from baybe_b200.nipv import NipvScorer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


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


def _events(fn, reps=20, warm=3) -> float:
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_times() -> list[dict]:
    out = []
    n, d, P = 256, 20, 10
    gp = _gp(n, d)
    rng = np.random.default_rng(1)
    x = torch.rand(P, d, device="cuda")
    for M in (4096, 65536, 1_000_000):
        sc = NipvScorer(gp, AcqConfig("qNIPV"), rng.uniform(0, 1, (M, d)))
        for Cn in (0, 8):
            c = sc.conditioned(rng.uniform(0, 1, (Cn, d)) if Cn else None, None)
            cond_x, beta = c.cond if c.linv is not None else (None, None)
            phi = lambda: torch.ops.baybe_b200.nipv_phi(sc.xm, c.cross_m, c.linv, gp.handle)  # noqa: E731
            img = phi()
            grad = lambda: torch.ops.baybe_b200.nipv_grad(x, img, M, cond_x, beta, c.linv, gp.handle)  # noqa: E731
            ms_phi, ms_grad = _events(phi), _events(grad)
            r = n + Cn
            tiles = math.ceil(P / 16)
            bytes_ = (r + d) * M * 4 * tiles
            out.append({"M": M, "C": Cn, "P": P, "nipv_phi_ms": ms_phi, "nipv_grad_ms": ms_grad,
                        "grad_GBps": bytes_ / (ms_grad * 1e-3) / 1e9,
                        "grad_share_of_hbm_bound": bytes_ / HBM_BYTES_PER_S / (ms_grad * 1e-3)})
    return out


def recommend_times() -> dict:
    res = {}
    d = 4
    gp = _gp(64, d, seed=2)
    xm = np.random.default_rng(4).uniform(0, 1, (4096, d))
    cb = np.array([np.zeros(d), np.ones(d)])
    for q in (1, 4):
        for warm in (True, False):
            sc = NipvScorer(gp, AcqConfig("qNIPV"), xm)
            cond_s = [0.0]
            conditioned, phi = sc.conditioned, nv._nipv_phi

            def timed(fn):
                def run(*a, **k):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    r = fn(*a, **k)
                    torch.cuda.synchronize()
                    cond_s[0] += time.perf_counter() - t0
                    return r
                return run

            sc.conditioned = timed(conditioned)
            nv._nipv_phi = timed(phi)
            try:
                st: dict = {}
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), cb, q, seed=1, stats=st)
                torch.cuda.synchronize()
                total = time.perf_counter() - t0
            finally:
                nv._nipv_phi = phi
            if warm:
                continue
            res[f"continuous_4d_q{q}"] = {"total_s": total, "conditioning_and_image_s": cond_s[0],
                                          "polish_s": st.get("polish_s", 0.0), "grad_calls": st.get("grad_calls", 0),
                                          "grad_s": st.get("grad_s", 0.0),
                                          "raw_sweep_and_scoring_s": total - st.get("polish_s", 0.0)}
    return res


def main() -> None:
    if not torch.cuda.is_available():
        raise SystemExit("bench_nipv_grad.py measures on a GPU; none found")
    info = _card()
    print(json.dumps({**info, "nipv_grad": kernel_times(), **recommend_times()}))


if __name__ == "__main__":
    main()
