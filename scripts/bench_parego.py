"""Candidates/s of qLogNParEGO on 1M x 20D, n = 256, S = 512, with 2 and 5 targets: one greedy round without pending
points (|C| = 1 on this workload) and one with 8 (|C| = 9).  Timed separately: the pruning of the 256-row baseline (one
bb_joint_posterior per target + 2048 float64 samples of the scalarisation on the host, host clock around a
synchronised call), the conditioning set-up of a round (host, float64, one bb_joint_posterior per target), the M
posterior passes with the cross covariance to C (bb_posterior) and bb_parego_score (CUDA events, L2 flushed untimed
before every step, SM clocks sampled with NVML).  Prints one JSON line; writes nothing."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from bench import ClockSampler  # noqa: E402
from baybe_b200 import DeviceGP, parego  # noqa: E402
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
    x = torch.from_numpy(w.candidates).to(dev, torch.float32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    cfg = AcqConfig(kind="qLogNParEGO")
    pend8 = w.candidates[np.random.default_rng(3).choice(args.N, 8, replace=False)]
    results = {}
    with ClockSampler(0) as clk:
        for M in (2, 5):
            kw = w.gp_kwargs()
            gps = [DeviceGP(device=dev, **{**kw, "train_y": smooth_target(w.train_x, seed=7 * m + 1)})
                   for m in range(M)]
            lam = np.full(M, 1.0 / M)
            a, b = np.ones(M), np.zeros(M)
            t_prune = []
            for step in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                scorer = parego.ParegoScorer(gps, cfg, a, b, w.train_x, lam)
                torch.cuda.synchronize()
                if step >= args.warmup:
                    t_prune.append((time.perf_counter() - t0) * 1e3)
            rounds = {}
            for name, pend in (("no_pending", None), ("pending_8", pend8)):
                P = 0 if pend is None else len(pend)
                z = scorer.base_samples(args.samples, P, seed=1234)
                t_setup, t_post, t_score = [], [], []
                for step in range(args.warmup + args.steps):
                    torch.cuda.synchronize()
                    h0 = time.perf_counter()
                    rows, linv, wv, g, _, conds = scorer.conditioning(pend, None, z.numpy())
                    t = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(dev, torch.float32)  # noqa: E731
                    linv_d, w_d, z_d, g_d = t(linv), t(wv.transpose(0, 2, 1)), t(z), t(g)
                    torch.cuda.synchronize()
                    h1 = time.perf_counter()
                    flush.fill_(1)
                    torch.cuda.synchronize()
                    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                    e[0].record()
                    post = [gp.cross_covariance(x, px, beta) for gp, (px, beta) in zip(gps, conds)]
                    mu = torch.stack([p[0] for p in post])
                    var = torch.stack([p[1] for p in post])
                    cross = torch.stack([p[2] for p in post])
                    e[1].record()
                    torch.ops.baybe_b200.parego_score(mu, var, cross, linv_d, w_d, z_d, g_d, None, None,
                                                      [float(v) for v in scorer.W], [float(v) for v in scorer.V],
                                                      [scorer.alpha, cfg.tau_relu, cfg.tau_max], 0, False)
                    e[2].record()
                    torch.cuda.synchronize()
                    if step >= args.warmup:
                        t_setup.append((h1 - h0) * 1e3)
                        t_post.append(e[0].elapsed_time(e[1]))
                        t_score.append(e[1].elapsed_time(e[2]))
                ts, tp, tn = statistics.median(t_setup), statistics.median(t_post), statistics.median(t_score)
                rounds[name] = {"n_conditioning": len(rows), "conditioning_setup_ms": round(ts, 4),
                                "posterior_cross_ms": round(tp, 4), "parego_score_ms": round(tn, 4),
                                "device_round_ms": round(tp + tn, 4),
                                "candidates_per_s": args.N / ((tp + tn) * 1e-3)}
            results[f"M{M}"] = {"kept_baseline": int(len(scorer.winners)),
                                "prune_ms": round(statistics.median(t_prune), 4), "rounds": rounds}
    props = torch.cuda.get_device_properties(dev)
    power = None
    try:
        import pynvml

        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    print(json.dumps({
        "workload": f"qLogNParEGO, M targets, N={args.N}, d=20, n=256 baseline rows, S={args.samples}",
        "gpu": props.name, "power_limit_w": power, "clocks": clk.summary(), "targets": results,
        "steps": args.steps, "warmup": args.warmup,
        "timing": "median over steps; device steps: L2 flushed (256 MiB write, untimed), CUDA events; host steps: "
                  "perf_counter around synchronised work",
    }))


if __name__ == "__main__":
    main()
