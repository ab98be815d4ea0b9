"""Candidates/s of qLogEHVI (Pareto objective, 2 targets) on 1M x 20D, n = 256, S = 512: one greedy round with no
pending points.  The two posterior passes (bb_posterior, one per target model) and bb_hvi_score are timed
separately with CUDA events, L2 flushed (untimed) before every step, SM clocks sampled with NVML.  Prints one JSON
line; writes nothing."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from bench import ClockSampler  # noqa: E402
from baybe_b200 import DeviceGP, multiobjective as mo  # noqa: E402
from baybe_b200.engine import AcqConfig  # noqa: E402
from baybe_b200.synthetic import numeric_grid_workload, smooth_target  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--samples", type=int, default=512)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    w = numeric_grid_workload(N=args.N, d=20, n=256, seed=0)
    y2 = smooth_target(w.train_x, seed=21) + 0.01 * np.random.default_rng(1).standard_normal(len(w.train_y))
    kw2 = dict(w.gp_kwargs(), train_y=y2)
    gps = [DeviceGP(device=dev, **w.gp_kwargs()), DeviceGP(device=dev, **kw2)]
    a, b = np.array([1.0, -1.0]), np.zeros(2)
    front = np.stack([gp.posterior(torch.from_numpy(w.train_x))[0].double().cpu().numpy() for gp in gps], 1) * a + b
    scorer = mo.HviScorer(gps, AcqConfig(kind="qLogEHVI"), a, b, mo.compute_ref_point(front), front)
    x = torch.from_numpy(w.candidates).to(dev, torch.float32)
    z = scorer.base_samples(args.samples, 0, seed=1234)
    lower, upper, counts, C = mo._padded([(scorer.lower, scorer.upper)], 2)
    cells = [torch.from_numpy(t).to(dev) for t in (lower, upper, counts)]
    zd = z.to(dev, torch.float32).contiguous()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def posterior():
        post = [gp.posterior(x) for gp in gps]
        return torch.stack([p[0] for p in post]), torch.stack([p[1] for p in post])

    def hvi(mu, var):
        return torch.ops.baybe_b200.hvi_score(mu, var, None, None, None, zd, *cells, None, 12, scorer.cfg.params(),
                                              list(a), list(b), 0, False)

    t_post, t_hvi = [], []
    with ClockSampler(0) as clk:
        for step in range(args.warmup + args.steps):
            flush.fill_(1)
            torch.cuda.synchronize()
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            mu, var = posterior()
            e[1].record()
            hvi(mu, var)
            e[2].record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                t_post.append(e[0].elapsed_time(e[1]))
                t_hvi.append(e[1].elapsed_time(e[2]))
    props = torch.cuda.get_device_properties(dev)
    power = None
    try:
        import pynvml

        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    tp, th = statistics.median(t_post), statistics.median(t_hvi)
    print(json.dumps({
        "workload": f"qLogEHVI, 2 targets, N={args.N}, d=20, n=256, S={args.samples}, no pending points",
        "gpu": props.name, "power_limit_w": power, "clocks": clk.summary(),
        "front_size": int(len(mo._pareto_points(front, scorer.ref))), "cells": int(C),
        "posterior_ms": round(tp, 4), "hvi_score_ms": round(th, 4), "round_ms": round(tp + th, 4),
        "candidates_per_s": args.N / ((tp + th) * 1e-3), "steps": args.steps, "warmup": args.warmup,
        "timing": "median over steps; per step L2 flushed (256 MiB write, untimed), CUDA events",
    }))


if __name__ == "__main__":
    main()
