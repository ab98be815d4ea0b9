"""Same-box A/B of ``bb_acq_grad_large`` and ``bb_objective_grad`` across library builds.
dump: the value and gradient of every oracle-comparison case of tests/test_gpu_acq_grad_large.py (families x shapes x
the 11 kinds, points on training rows, 1, 8 and 31 pending points, the d100_n200 wide model with and without pending
points) and of tests/test_gpu_objective_continuous.py (its CASES), then the per-call times.
time: the per-call times only -- the median of 20 CUDA-event-timed calls after 3 warm-up calls of qLogEI, S = 512,
10^4 points, p in {0, 8}, for bb_acq_grad_large at n = 256, d = 8 and for bb_objective_grad on a GEOM_MEAN of two
targets at n = 256, d = 8.
usage: BB_LIB_VARIANT=<name> python scripts/ab_objective_grad.py dump <file.pt>   (no variable: the current build)
       BB_LIB_VARIANT=<name> python scripts/ab_objective_grad.py time
       python scripts/ab_objective_grad.py compare <a.pt> <b.pt>                 (bit-for-bit; exit status 1 on a difference)"""
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402


def _acq_grad_large_cases(out: dict) -> None:
    from baybe_b200 import sobol_normal_samples
    from baybe_b200._lib import GRAD_KINDS
    from tests.test_gpu_acq_grad_large import FAMILIES, MC, S, SHAPES, _acq, _setup, _wide_d100

    def kinds(tag, gp, om, X, pts, z, ks, pend=None):
        for kind in ks:
            _, cfg = _acq(kind, om, X)
            v, g = gp.value_and_grad(cfg, torch.from_numpy(pts), z if cfg.is_mc else None, pend)
            out[f"acq_grad_large-{tag}-{kind}"] = (v.cpu(), g.cpu())

    z1 = sobol_normal_samples(S, 1, 7)
    for family in FAMILIES:
        for d, n, os_ in SHAPES:
            gp, om, X, pts = _setup(family, d, n, os_)
            kinds(f"{family}-d{d}-n{n}", gp, om, X, pts, z1, GRAD_KINDS)
    for family in ("matern32", "matern52", "rbf"):
        for n in (320, 1000):
            gp, om, X, _ = _setup(family, 4, n, 1.3, seed=2)
            kinds(f"{family}-rows-n{n}", gp, om, X, np.vstack([X[:8], X[n // 2 : n // 2 + 4]]), z1, GRAD_KINDS)
    for family in ("matern52", "rbf"):
        for p in (1, 8, 31):
            gp, om, X, pts = _setup(family, 4, 400, 1.3, seed=p)
            rng = np.random.default_rng(100 + p)
            pend = np.vstack([rng.uniform(0, 1, (p - 1, 4)), pts[:1] + 0.02]).clip(0, 1) if p > 1 else pts[:1] + 0.02
            kinds(f"{family}-p{p}", gp, om, X, pts, sobol_normal_samples(S, 1 + p, 11), MC, pend)
    w, gp, om = _wide_d100()
    rng = np.random.default_rng(5)
    pts = np.vstack([w.candidates[:10], w.train_x[:4] + 0.02 * rng.normal(size=(4, 100))]).clip(0, 1)
    kinds("d100_n200", gp, om, w.train_x, pts, z1, GRAD_KINDS)
    for p in (1, 8, 31):
        kinds(f"d100_n200-p{p}", gp, om, w.train_x, w.candidates[:8], sobol_normal_samples(S, 1 + p, 13),
              ("qLogEI", "qEI", "qUCB"), w.candidates[100 : 100 + p])


def _objective_grad_cases(out: dict) -> None:
    from tests.test_gpu_objective_continuous import CASES, PROGRAMS, _inputs, _Pair, _scorer

    for name, kind, scal, progs, fam, ns, os_, P in CASES:
        pairs = [_Pair(fam, n, os_, seed=m) for m, n in enumerate(ns)]
        M = len(pairs)
        weights = [1.0] if M == 1 else list(np.linspace(1.0, 2.0, M) / np.linspace(1.0, 2.0, M).sum())
        if scal == "GEOM_MEAN":
            progs = ["bell" if p in ("minimised", "log_exp", "two_sided", "pow", "clamp") else p for p in progs]
        sc = _scorer(pairs, kind, scal, [PROGRAMS[p] for p in progs], weights)
        pts, pend, z = _inputs(sc, P)
        v, g = sc.value_and_grad(torch.from_numpy(pts), pend, z)
        out[f"objective_grad-{name}"] = (v.cpu(), g.cpu())


def times() -> dict:
    from baybe_b200 import AcqConfig, sobol_normal_samples
    from scripts.bench_acq_grad_large import _gp
    from scripts.bench_objective_grad import _events, _gps, _scorer

    res = {}
    gp = _gp(256, 8)
    cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
    sc = _scorer(_gps(2, 256, 8))
    x = torch.rand(10_000, 8, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    for p in (0, 8):
        pend = np.random.default_rng(1).uniform(0, 1, (p, 8)) if p else None
        z = sobol_normal_samples(512, 1 + p, 3)
        res[f"acq_grad_large_n256_p{p}"] = _events(lambda: gp.value_and_grad(cfg, x, z, pend))
        zo = sc.base_samples(512, p, 0)
        res[f"objective_grad_n256_M2_p{p}"] = _events(lambda: sc.value_and_grad(x, pend, zo))
    return res


def dump(path: str) -> None:
    out: dict = {}
    _acq_grad_large_cases(out)
    _objective_grad_cases(out)
    torch.save(out, path)
    t = times()
    print(f"variant {os.environ.get('BB_LIB_VARIANT', 'current')}: {len(out)} cases, ms per call (10^4 points) "
          + ", ".join(f"{k} {v:.4f}" for k, v in t.items()), flush=True)


def compare(a: str, b: str) -> int:
    A, B = torch.load(a), torch.load(b)
    assert A.keys() == B.keys()
    bad = [k for k in A if not (torch.equal(A[k][0], B[k][0]) and torch.equal(A[k][1], B[k][1]))]
    for prefix in ("acq_grad_large-", "objective_grad-"):
        keys = [k for k in A if k.startswith(prefix)]
        print(f"{prefix[:-1]}: {sum(k not in bad for k in keys)} of {len(keys)} cases bit-identical")
    if bad:
        print(f"differ: {bad}")
    return 1 if bad else 0


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2])
    elif sys.argv[1] == "time":
        print(f"variant {os.environ.get('BB_LIB_VARIANT', 'current')}: ms per call (10^4 points) "
              + ", ".join(f"{k} {v:.4f}" for k, v in times().items()), flush=True)
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
