"""Same-box A/B of ``bb_acq_grad`` across library builds: the value and gradient of every case of
tests/test_gpu_continuous.py's oracle comparisons (4 families x 3 shapes x 11 kinds without pending points; Matern-5/2
and RBF with 1, 8 and 31 pending points x the 5 Monte Carlo kinds), and the median per-call time (CUDA events, 20 calls
after 3 warm-up calls) at n = 256, d = 8, qLogEI, S = 512, 10^4 points, p in {0, 8}.
usage: BB_LIB_VARIANT=<name> python scripts/ab_acq_grad.py dump <file.pt>   (no variable: the current build)
       python scripts/ab_acq_grad.py compare <a.pt> <b.pt>                 (bit-for-bit; exit status 1 on a difference)"""
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402


def dump(path: str) -> None:
    from baybe_b200 import AcqConfig, sobol_normal_samples
    from baybe_b200._lib import GRAD_KINDS
    from scripts.bench_continuous import _gp
    from scripts.bench_objective_grad import _events
    from tests.test_gpu_continuous import FAMILIES, MC, S, SHAPES, _acq, _setup

    out = {}
    for family in FAMILIES:
        for d, n, os_ in SHAPES:
            gp, om, X, pts = _setup(family, d, n, os_)
            z = sobol_normal_samples(S, 1, 7)
            for kind in GRAD_KINDS:
                _, cfg = _acq(kind, om, X)
                v, g = gp.value_and_grad(cfg, torch.from_numpy(pts), z if cfg.is_mc else None)
                out[f"{family}-d{d}-n{n}-{kind}"] = (v.cpu(), g.cpu())
    for family in ("matern52", "rbf"):
        for p in (1, 8, 31):
            gp, om, X, pts = _setup(family, 4, 64, 1.3, seed=p)
            rng = np.random.default_rng(100 + p)
            pend = np.vstack([rng.uniform(0, 1, (p - 1, 4)), pts[:1] + 0.02]).clip(0, 1) if p > 1 else pts[:1] + 0.02
            z = sobol_normal_samples(S, 1 + p, 11)
            for kind in MC:
                _, cfg = _acq(kind, om, X)
                v, g = gp.value_and_grad(cfg, torch.from_numpy(pts), z, pend)
                out[f"{family}-p{p}-{kind}"] = (v.cpu(), g.cpu())
    times = {}
    gp = _gp(256, 8)
    cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
    x = torch.rand(10_000, 8, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    for p in (0, 8):
        pend = np.random.default_rng(1).uniform(0, 1, (p, 8)) if p else None
        z = sobol_normal_samples(512, 1 + p, 3)
        times[f"p{p}"] = _events(lambda: gp.value_and_grad(cfg, x, z, pend))
    torch.save(out, path)
    print(f"variant {os.environ.get('BB_LIB_VARIANT', 'current')}: {len(out)} cases, ms per call (10^4 points) "
          + ", ".join(f"{k} {v:.4f}" for k, v in times.items()), flush=True)


def compare(a: str, b: str) -> int:
    A, B = torch.load(a), torch.load(b)
    assert A.keys() == B.keys()
    bad = [k for k in A if not (torch.equal(A[k][0], B[k][0]) and torch.equal(A[k][1], B[k][1]))]
    print(f"{len(A) - len(bad)} of {len(A)} cases bit-identical" + (f"; differ: {bad}" if bad else ""))
    return 1 if bad else 0


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2])
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
