"""Candidates/s of qLogNEI on 1M x 20D, n = 256, S = 512: one greedy round without pending points and one with 8.
Timed separately: the pruning of the 256-row baseline (bb_joint_posterior + 2048 float64 samples on the host, one
per scorer, host clock around a synchronised call), the conditioning set-up of a round (host, float64), the
posterior pass with the cross covariance to C (bb_posterior) and bb_nei_score (CUDA events, L2 flushed untimed before
every step, SM clocks sampled with NVML).  Prints one JSON line; writes nothing."""
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
from baybe_b200 import DeviceGP, noisy  # noqa: E402
from baybe_b200.engine import AcqConfig  # noqa: E402
from baybe_b200.synthetic import numeric_grid_workload  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--samples", type=int, default=512)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    w = numeric_grid_workload(N=args.N, d=20, n=256, seed=0)
    gp = DeviceGP(device=dev, **w.gp_kwargs())
    cfg = AcqConfig(kind="qLogNEI")
    x = torch.from_numpy(w.candidates).to(dev, torch.float32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    t_prune = []
    for step in range(args.warmup + args.steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        scorer = noisy.NeiScorer(gp, cfg, w.train_x)
        torch.cuda.synchronize()
        if step >= args.warmup:
            t_prune.append((time.perf_counter() - t0) * 1e3)

    pend8 = w.candidates[np.random.default_rng(3).choice(args.N, 8, replace=False)]
    rounds = {}
    with ClockSampler(0) as clk:
        for name, pend in (("no_pending", None), ("pending_8", pend8)):
            P = 0 if pend is None else len(pend)
            z = scorer.base_samples(args.samples, P, seed=1234)
            t_setup, t_post, t_nei = [], [], []
            for step in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                h0 = time.perf_counter()
                rows, linv, wv, g, _, (px, beta) = scorer.conditioning(pend, None, z.numpy())
                t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, torch.float32)  # noqa: E731
                linv_d, w_d, z_d, g_d = t(linv), t(wv.T), t(z), t(g)
                torch.cuda.synchronize()
                h1 = time.perf_counter()
                flush.fill_(1)
                torch.cuda.synchronize()
                e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                e[0].record()
                mu, var, cross = gp.cross_covariance(x, px, beta)
                e[1].record()
                torch.ops.baybe_b200.nei_score(mu, var, cross, linv_d, w_d, z_d, g_d, None, None, True,
                                               [cfg.obj_scale, cfg.obj_shift, cfg.tau_relu, cfg.tau_max], 0, False)
                e[2].record()
                torch.cuda.synchronize()
                if step >= args.warmup:
                    t_setup.append((h1 - h0) * 1e3)
                    t_post.append(e[0].elapsed_time(e[1]))
                    t_nei.append(e[1].elapsed_time(e[2]))
            ts, tp, tn = statistics.median(t_setup), statistics.median(t_post), statistics.median(t_nei)
            rounds[name] = {"n_conditioning": len(rows), "conditioning_setup_ms": round(ts, 4),
                            "posterior_cross_ms": round(tp, 4), "nei_score_ms": round(tn, 4),
                            "device_round_ms": round(tp + tn, 4), "candidates_per_s": args.N / ((tp + tn) * 1e-3)}
    props = torch.cuda.get_device_properties(dev)
    power = None
    try:
        import pynvml

        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    print(json.dumps({
        "workload": f"qLogNEI, one affine target, N={args.N}, d=20, n=256 baseline rows, S={args.samples}",
        "gpu": props.name, "power_limit_w": power, "clocks": clk.summary(),
        "kept_baseline": int(len(scorer.winners)), "prune_ms": round(statistics.median(t_prune), 4),
        "rounds": rounds, "steps": args.steps, "warmup": args.warmup,
        "timing": "median over steps; device steps: L2 flushed (256 MiB write, untimed), CUDA events; host steps: "
                  "perf_counter around synchronised work",
    }))


if __name__ == "__main__":
    main()
