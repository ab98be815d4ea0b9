"""Candidates/s of qLogEI with a two-target GEOM_MEAN desirability objective on 1M x 20D, n = 256, S = 512: one greedy
round with no pending points.  Targets: `clamp().normalize()` and `match_triangular`, compiled as
baybe_b200.objectives does.  The two posterior passes (bb_posterior, one per target model) and bb_objective_score are
timed separately with CUDA events, L2 flushed (untimed) before every step, SM clocks sampled with NVML.  Prints one
JSON line; writes nothing."""
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
from baybe_b200 import DeviceGP, _lib, objectives as ob  # noqa: E402
from baybe_b200.engine import AcqConfig  # noqa: E402
from baybe_b200.synthetic import numeric_grid_workload, smooth_target  # noqa: E402

# NumericalTarget("t0").clamp(-1, 1).normalize() and NumericalTarget.match_triangular("t1", cutoffs=(-1, 1)),
# in compiled form
PROGRAMS = [[("CLAMP", (-1.0, 1.0, 0.0)), ("AFFINE", (0.5, 0.5, 0.0))],
            [("TWO_SIDED", (1.0, -1.0, 0.0)), ("AFFINE", (1.0, 1.0, 0.0)), ("CLAMP", (0.0, float("inf"), 0.0))]]


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
    comp = ob.CompiledObjective(["t0", "t1"], PROGRAMS, "GEOM_MEAN", [0.5, 0.5])
    means = np.stack([gp.posterior(torch.from_numpy(w.train_x))[0].double().cpu().numpy() for gp in gps], 1)
    cfg = AcqConfig(kind="qLogEI", best_f=float(np.max(ob.evaluate_objective(comp, means))))
    x = torch.from_numpy(w.candidates).to(dev, torch.float32)
    z = ob.ObjectiveScorer(gps, cfg, comp).base_samples(args.samples, 0, seed=1234)
    zd = z.to(dev, torch.float32).contiguous()
    ops, prm, n_ops = comp.flat()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def posterior():
        post = [gp.posterior(x) for gp in gps]
        return torch.stack([p[0] for p in post]), torch.stack([p[1] for p in post])

    def score(mu, var):
        return torch.ops.baybe_b200.objective_score(mu, var, None, None, None, None, zd, None, _lib.ACQ_KIND["qLogEI"],
                                                    cfg.params(), _lib.OBJ_SCALARIZER["GEOM_MEAN"], ops, prm, n_ops,
                                                    [0.5, 0.5], 0, False)

    t_post, t_obj = [], []
    with ClockSampler(0) as clk:
        for step in range(args.warmup + args.steps):
            flush.fill_(1)
            torch.cuda.synchronize()
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            mu, var = posterior()
            e[1].record()
            score(mu, var)
            e[2].record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                t_post.append(e[0].elapsed_time(e[1]))
                t_obj.append(e[1].elapsed_time(e[2]))
    props = torch.cuda.get_device_properties(dev)
    power = None
    try:
        import pynvml

        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    tp, to = statistics.median(t_post), statistics.median(t_obj)
    print(json.dumps({
        "workload": f"qLogEI, GEOM_MEAN desirability of 2 targets (clamp-normalised, triangular), N={args.N}, d=20, "
                    f"n=256, S={args.samples}, no pending points",
        "gpu": props.name, "power_limit_w": power, "clocks": clk.summary(),
        "posterior_ms": round(tp, 4), "objective_score_ms": round(to, 4), "round_ms": round(tp + to, 4),
        "candidates_per_s": args.N / ((tp + to) * 1e-3), "steps": args.steps, "warmup": args.warmup,
        "timing": "median over steps; per step L2 flushed (256 MiB write, untimed), CUDA events",
    }))


if __name__ == "__main__":
    main()
