"""qNIPV round on the device: 1M x 20D candidates, n = 256, M in {4096, 65536, 1M (the default fraction)} integration
points, each with |C| in {0, 8} conditioning points.  Per run: host conditioning, the two posterior passes and
bb_nipv_score (CUDA events), pairs/s and the achieved tensor-core rate (3 fp16 MMAs of r_pad per pair), and a
comparison leg: the same IVR from a chunked torch float32 composition (kernel matrix of the integration points
against the candidates, minus the phi product, squared and summed) on the same card, with the largest difference.

    python scripts/bench_nipv.py [--n-cand 1000000] [--legs 4096,65536,0]
Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from baybe_b200 import DeviceGP  # noqa: E402
from baybe_b200 import nipv  # noqa: E402
from baybe_b200.engine import AcqConfig  # noqa: E402
from baybe_b200.synthetic import numeric_grid_workload  # noqa: E402


def _torch_ivr(gp, X, XM, C_rows):
    """IVR of the rows of X in float32 torch: phi = L^-1 k(X_train, .) (+ L_C^-1 k_D(C, .)), then per chunk of
    integration points k(m, x) - phi_m . phi_x, squared and summed; original units."""
    tx = torch.from_numpy(gp.train_x).to(X.device, torch.float32)
    lo = torch.zeros(X.shape[1], device=X.device)
    ls = torch.from_numpy(np.asarray(gp.lengthscale, dtype=np.float32)).to(X.device)
    scale = float(gp.outputscale or 1.0)
    ys2 = float(gp.model.y_std) ** 2
    noise = max(float(gp.noise[0]), 1e-4)

    def k(a, b):  # Matern-5/2 on the [0,1]-normalised rows
        r = torch.cdist((a - lo) / ls, (b - lo) / ls)
        s = math.sqrt(5.0) * r
        return scale * (1 + s + s * s / 3) * torch.exp(-s)

    Kt = k(tx, tx) + noise * torch.eye(len(tx), device=X.device)
    Linv = torch.linalg.inv(torch.linalg.cholesky(Kt.double())).float()
    phi = lambda A: (Linv @ k(tx, A))  # noqa: E731  [n, rows]
    px = phi(X)
    kxx = scale - (px * px).sum(0)
    extra_x = extra_m = None
    if len(C_rows):
        pc = phi(C_rows)
        Kdc = k(C_rows, C_rows) - pc.T @ pc + noise * torch.eye(len(C_rows), device=X.device)
        Lc = torch.linalg.inv(torch.linalg.cholesky(Kdc.double())).float()
        extra_x = Lc @ (k(C_rows, X) - pc.T @ px)
        kxx = kxx - (extra_x * extra_x).sum(0)
    num = torch.zeros(len(X), device=X.device)
    chunk = max(256, (1 << 30) // len(X))  # a few [chunk, N] float32 temporaries of 4 GB at most
    for m0 in range(0, len(XM), chunk):
        A = XM[m0:m0 + chunk]
        pa = phi(A)
        G = k(A, X) - pa.T @ px
        if extra_x is not None:
            extra_m = Lc @ (k(C_rows, A) - pc.T @ pa)
            G = G - extra_m.T @ extra_x
        num += (G * G).sum(0)
    return num / (kxx + noise) * ys2


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-cand", type=int, default=1_000_000)
    ap.add_argument("--legs", default="4096,65536,0", help="integration point counts; 0 = all candidates")
    ap.add_argument("--conds", default="0,8")
    ap.add_argument("--torch-leg-max", type=int, default=1_000_000_000_000, help="skip the torch leg above M*N")
    args = ap.parse_args()
    from bench import ClockSampler

    dev = torch.device("cuda", 0)
    w = numeric_grid_workload(N=args.n_cand, d=20, n=256, seed=0)
    gp = DeviceGP(device=dev, **w.gp_kwargs())
    X = torch.from_numpy(w.candidates).to(dev, torch.float32).contiguous()
    rng = np.random.default_rng(0)
    props = torch.cuda.get_device_properties(dev)
    out = {"card": props.name, "N": args.n_cand, "d": 20, "n": 256, "runs": []}
    try:
        import subprocess

        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip()
        out["power_limit_and_max_sm_clock"] = q
    except OSError:
        pass
    with ClockSampler(0) as clocks:
        _runs(args, w, gp, X, rng, dev, out)
    out["clocks"] = clocks.summary()
    print(json.dumps(out))


def _runs(args, w, gp, X, rng, dev, out) -> None:
    for M in [int(v) for v in args.legs.split(",")]:
        M = M or args.n_cand
        XM = w.candidates[rng.choice(args.n_cand, M, replace=False)] if M < args.n_cand else w.candidates
        sc = nipv.NipvScorer(gp, AcqConfig(kind="qNIPV"), XM)
        for C in [int(v) for v in args.conds.split(",")]:
            pend = w.candidates[rng.choice(args.n_cand, C, replace=False)] if C else None
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows, linv, cond = sc.conditioning(pend, None)
            t_cond = time.perf_counter() - t0
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            if C:
                _, var, cx = gp.cross_covariance(X, *cond)
                _, var_m, cm = gp.cross_covariance(sc.xm, *cond)
                ld = torch.from_numpy(linv).to(dev, torch.float32).contiguous()
            else:
                _, var = gp.posterior(X)
                _, var_m = gp.posterior(sc.xm)
                cx = cm = ld = None
            ev[1].record()
            s, key = nipv._nipv_score(X, sc.xm, var.contiguous(), None if cx is None else cx.contiguous(),
                                      None if cm is None else cm.contiguous(), ld, None, gp.handle, 0, True)
            ev[2].record()
            torch.cuda.synchronize()
            t_post = ev[0].elapsed_time(ev[1]) / 1e3
            t_k = ev[1].elapsed_time(ev[2]) / 1e3
            pairs = float(args.n_cand) * M
            r_pad = -(-(256 + C) // 64) * 64
            run = {"M": M, "C": C, "host_conditioning_s": t_cond, "posterior_passes_s": t_post,
                   "nipv_score_s": t_k, "pairs_per_s": pairs / t_k,
                   "tensor_core_tflops": pairs * 3 * 2 * r_pad / t_k / 1e12}
            if pairs <= args.torch_leg_max:
                Ct = torch.from_numpy(np.asarray(rows, dtype=np.float32)).to(dev) if C else torch.zeros(0, 20,
                                                                                                       device=dev)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ref = _torch_ivr(gp, X, sc.xm, Ct)
                torch.cuda.synchronize()
                run["torch_f32_s"] = time.perf_counter() - t0
                run["max_abs_diff_vs_torch"] = float((ref - s).abs().max())
                run["max_ivr"] = float(s.max())
            out["runs"].append(run)
            print(json.dumps(run), file=sys.stderr, flush=True)


if __name__ == "__main__":
    main()
