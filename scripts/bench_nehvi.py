"""qNEHVI on 1M x 20D, n = 256, S = 512, with 2 and 3 targets: one greedy round without pending points and one with 8.
Timed separately: the pruning of the 256-row baseline (one bb_joint_posterior per target + 2048 float64 joint samples
and their Pareto masks on the host, host clock around synchronised work), the host sampling of the conditioning set
C (float64, one bb_joint_posterior per target), the S device decompositions of the sampled fronts (bb_hvi_decompose,
the copy of the points included), the M posterior passes with the cross covariance to C (bb_posterior) and
bb_hvi_score (CUDA events, L2 flushed untimed before every device step, SM clocks sampled with NVML).  Also times
bb_hvi_decompose for S = 512 sets of 31 normal points at M = 3 and 4 against box_decomposition on the host (a subset of
the samples, scaled to 512).  Prints one JSON line; writes nothing."""
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
from baybe_b200 import DeviceGP, nehvi  # noqa: E402
from baybe_b200 import multiobjective as mo  # noqa: E402
from baybe_b200.engine import AcqConfig  # noqa: E402
from baybe_b200.synthetic import numeric_grid_workload, smooth_target  # noqa: E402


def _events(k):
    return [torch.cuda.Event(enable_timing=True) for _ in range(k)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--samples", type=int, default=512)
    ap.add_argument("--host-samples", type=int, default=32, help="host decompositions timed (scaled to --samples)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    w = numeric_grid_workload(N=args.N, d=20, n=256, seed=0)
    x = torch.from_numpy(w.candidates).to(dev, torch.float32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    cfg = AcqConfig(kind="qNEHVI")
    pend8 = w.candidates[np.random.default_rng(3).choice(args.N, 8, replace=False)]
    results = {}
    with ClockSampler(0) as clk:
        for M in (2, 3):
            ys = np.stack([smooth_target(w.train_x, seed=7 * m + 1) for m in range(M)], 1)
            kw = w.gp_kwargs()
            gps = [DeviceGP(device=dev, **{**kw, "train_y": ys[:, m]}) for m in range(M)]
            a, b = np.ones(M), np.zeros(M)
            ref = mo.compute_ref_point(ys)
            t_prune = []
            for step in range(max(1, args.warmup // 2) + max(3, args.steps // 3)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                scorer = nehvi.NehviScorer(gps, cfg, a, b, ref, w.train_x)
                torch.cuda.synchronize()
                if step >= max(1, args.warmup // 2):
                    t_prune.append((time.perf_counter() - t0) * 1e3)
            rounds = {}
            for name, pend in (("no_pending", None), ("pending_8", pend8)):
                P = 0 if pend is None else len(pend)
                z = scorer.base_samples(args.samples, P, seed=1234)
                t_setup, t_dec, t_post, t_score = [], [], [], []
                for step in range(args.warmup + args.steps):
                    torch.cuda.synchronize()
                    h0 = time.perf_counter()
                    rows, linv, wv, o, conds = scorer.conditioning(pend, None, z.numpy())
                    linv_d = torch.from_numpy(linv).to(dev, torch.float32)
                    w_d = torch.from_numpy(wv).to(dev, torch.float32)
                    z_d = z.to(dev, torch.float32)
                    torch.cuda.synchronize()
                    h1 = time.perf_counter()
                    flush.fill_(1)
                    torch.cuda.synchronize()
                    e = _events(4)
                    e[0].record()
                    lower, upper, n_cells, _ = nehvi._hvi_decompose(o, scorer.ref, dev)
                    e[1].record()
                    post = [gp.cross_covariance(x, px, beta) for gp, (px, beta) in zip(gps, conds)]
                    mu = torch.stack([p[0] for p in post])
                    var = torch.stack([p[1] for p in post])
                    cross = torch.stack([p[2] for p in post])
                    e[2].record()
                    torch.ops.baybe_b200.hvi_score(mu, var, cross, linv_d, w_d, z_d, lower, upper, n_cells, None,
                                                   11, AcqConfig(kind="qEHVI").params(), [float(v) for v in a],
                                                   [float(v) for v in b], 0, False)
                    e[3].record()
                    torch.cuda.synchronize()
                    if step >= args.warmup:
                        t_setup.append((h1 - h0) * 1e3)
                        t_dec.append(e[0].elapsed_time(e[1]))
                        t_post.append(e[1].elapsed_time(e[2]))
                        t_score.append(e[2].elapsed_time(e[3]))
                ts, td, tp, tn = (statistics.median(v) for v in (t_setup, t_dec, t_post, t_score))
                rounds[name] = {"n_conditioning": len(rows), "max_cells": int(n_cells.max()),
                                "host_sampling_of_C_ms": round(ts, 4), "device_decompositions_ms": round(td, 4),
                                "posterior_cross_ms": round(tp, 4), "hvi_score_ms": round(tn, 4),
                                "round_ms": round(ts + td + tp + tn, 4),
                                "candidates_per_s": args.N / ((ts + td + tp + tn) * 1e-3)}
            results[f"M{M}"] = {"kept_baseline": int(len(scorer.winners)),
                                "prune_ms": round(statistics.median(t_prune), 4), "rounds": rounds}
        decomp = {}
        for M in (3, 4):
            pts = np.random.default_rng(M).normal(size=(args.samples, 31, M))
            ref = np.full(M, -2.0)
            t_dev = []
            for step in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                e = _events(2)
                p_d = torch.from_numpy(pts.astype(np.float32)).to(dev)
                e[0].record()
                _, _, cnt, _ = torch.ops.baybe_b200.hvi_decompose(p_d, None, [float(r) for r in ref], 1024)
                e[1].record()
                torch.cuda.synchronize()
                if step >= args.warmup:
                    t_dev.append(e[0].elapsed_time(e[1]))
            k = min(args.host_samples, args.samples)
            t0 = time.perf_counter()
            for s in range(k):
                mo.box_decomposition(pts[s].astype(np.float32).astype(np.float64), ref)
            t_host = (time.perf_counter() - t0) * 1e3 * args.samples / k
            decomp[f"M{M}"] = {"points": 31, "S": args.samples, "max_cells": int(cnt.max()),
                               "device_ms": round(statistics.median(t_dev), 4),
                               "host_loop_ms_scaled": round(t_host, 1), "host_samples_timed": k}
    props = torch.cuda.get_device_properties(dev)
    power = None
    try:
        import pynvml

        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    print(json.dumps({
        "workload": f"qNEHVI, M targets, N={args.N}, d=20, n=256 baseline rows, S={args.samples}",
        "gpu": props.name, "power_limit_w": power, "clocks": clk.summary(), "targets": results,
        "decompose_31_points": decomp, "steps": args.steps, "warmup": args.warmup,
        "timing": "median over steps; device steps: L2 flushed (256 MiB write, untimed), CUDA events; host steps: "
                  "perf_counter around synchronised work",
    }))


if __name__ == "__main__":
    main()
