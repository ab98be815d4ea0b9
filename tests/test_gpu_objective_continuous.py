"""GPU tests of ``bb_objective_grad``: value and gradient against float64 autograd of the literal definition
(tests/objective_grad_oracle.py), the value against ``ObjectiveScorer.scores`` (``bb_objective_score``), determinism,
the optimiser's quality with a match target, and Campaign flows on the engine.

Gradient bound, per row i and column j (tests/test_gpu_continuous.py's bound, summed over the targets m):

    |g_ij - g_ref,ij| <= 1e-3 |g_ref,ij| + 1e-7 max_m s_y,m
        + sum_m EPS32_m * (|A_mu,m| T_mu,m + |A_var,m| T_var,m + sum_p |A_c,mp| T_c,mp)_j
        + sum_m sum over the partials A of max_corner |A(mu_m +- dmu_m, var_m +- dvar_m) - A| * |d moment / dx_j|
        + KINK_i,

with A_mu,m, A_var,m, A_c,mp the float64 partial derivatives of the value with respect to target m's moments, dmu /
dvar the stated posterior tolerances of tests/helpers.py, T the sums of absolute terms the device adds in fp32 and
EPS32 = 2^-19 sqrt(n_m).  KINK_i allows for the samples the oracle finds within roundoff of a kink of the objective
(a CLAMP bound or TWO_SIDED midpoint of a program, or o = best_f for qEI): fp32 may put such a sample on the other
side, which moves the gradient by |jump| / S; the jump is taken as 2 max_j |g_ref,ij| (a sample's contribution
changing sign at the scale of the whole gradient), so KINK_i = n_kink,i * 2 max_j |g_ref,ij| / S.  Samples within
1e-4 (1 + |kink|) of a kink count.  The value must agree with bb_objective_score's within 2e-4 + 1e-4 |value| plus
1.5 times the first-order change the stated posterior tolerances can cause (the two compute the moments on different
fp32 paths)."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import AcqConfig, DeviceGP
from baybe_b200.objectives import CompiledObjective, ObjectiveScorer
from oracle import reference_path as rp
from tests.continuous_oracle import oracle_moments
from tests.helpers import posterior_tolerances
from tests.objective_grad_oracle import objective_grad_f64, objective_value

pytestmark = pytest.mark.gpu

FAMILIES = ("matern12", "matern32", "matern52", "rbf")
MC = ("qLogEI", "qEI", "qUCB", "qSR", "qPI")
ANALYTIC = ("EI", "LogEI", "PI", "UCB", "PM", "PSTD")
S = 128
D = 3


class _Pair:
    """A device model and its oracle (``.om``, what the float64 stand-in reads)."""

    def __init__(self, family, n, outputscale, seed):
        rng = np.random.default_rng(seed)
        X = rng.uniform(0, 1, (n, D))
        y = np.sin(3 * X[:, 0]) + X[:, 1] ** 2 + 0.3 * seed + 0.05 * rng.normal(size=n)
        ls = np.array([0.45, 0.6, 0.0])  # one inactive column
        bounds = np.array([np.zeros(D), np.ones(D)])
        self.gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=bounds, family=family, lengthscale=ls,
                           noise=1e-2, outputscale=outputscale)
        spec = oracle.KernelSpec(family=family, lengthscale=ls[:2], active_dims=[0, 1], outputscale=outputscale)
        self.om = oracle.build_model(spec, X, y, bounds, noise=1e-2)
        self.X = X


# programs over raw y (targets around 0..2): every opcode, and nested composites
PROGRAMS = {
    "affine": [("AFFINE", (0.8, 0.1, 0.0))],
    "minimised": [("AFFINE", (-1.0, 0.0, 0.0))],
    "const": [("CONST", (0.4, 0.0, 0.0))],
    "clamp": [("CLAMP", (-0.3, 1.1, 0.0))],
    "two_sided": [("TWO_SIDED", (-0.7, 1.3, 0.6, ))],
    "bell": [("BELL", (0.9, 0.6, 0.0))],
    "log_exp": [("EXP", (0.0, 0.0, 0.0)), ("LOG", (0.0, 0.0, 0.0))],
    "pow": [("AFFINE", (0.5, 1.0, 0.0)), ("POW_INT", (3.0, 0.0, 0.0))],
    "sigmoid": [("SIGMOID", (0.7, -2.5, 0.0))],
    "add_mul": [("BELL", (0.5, 0.8, 0.0)), ("DUP_INPUT", (0.0, 0.0, 0.0)), ("SIGMOID", (1.0, -3.0, 0.0)),
                ("DUP_INPUT", (0.0, 0.0, 0.0)), ("AFFINE", (0.5, 0.2, 0.0)), ("MUL", (0.0, 0.0, 0.0)),
                ("ADD", (0.0, 0.0, 0.0))],
}
for _p in PROGRAMS.values():
    for _i, (_o, _a) in enumerate(_p):
        _p[_i] = (_o, tuple(_a) + (0.0,) * (3 - len(_a)))


def _scorer(pairs, kind, scal, progs, weights, beta=0.6):
    comp = CompiledObjective([f"t{m}" for m in range(len(pairs))], progs, scal, weights)
    analytic = None if kind in MC else comp
    cfg = AcqConfig(kind, best_f=0.0, beta=beta)
    sc = ObjectiveScorer([p.gp for p in pairs], cfg, comp, analytic)
    # best_f as the reference forms it: the objective of the posterior means at the first model's training inputs
    from baybe_b200.objectives import evaluate_objective

    means = np.stack([oracle.posterior(p.om, pairs[0].X)[0].numpy() for p in pairs], 1)
    sc.cfg = AcqConfig(kind, best_f=float(np.max(evaluate_objective(comp, means))), beta=beta)
    return sc


def _inputs(sc, P, seed=0):
    rng = np.random.default_rng(seed + 7)
    pts = rng.uniform(0.05, 0.95, (10, D))
    pend = rng.uniform(0, 1, (P, D)) if P else None
    z = sc.base_samples(S, P, seed) if sc.cfg.is_mc else None
    return pts, pend, z


def _oracle(sc, pairs, pts, pend, z):
    P, stats, linv, w, terms, zd = sc.conditioning(pend, z)
    kc = sc.kernel_comp
    ops, args, n_ops = kc.flat()
    from baybe_b200 import _lib

    a = (pts, None if pend is None else pend, None, linv, w, terms, zd, _lib.ACQ_KIND[sc.cfg.kind], sc.cfg.params(),
         _lib.OBJ_SCALARIZER[kc.scalarizer], ops, args, n_ops, [float(v) for v in kc.weights])
    val, g = objective_grad_f64(pairs, *a)
    return val.double(), g.double(), (linv, w, terms, zd, kc)


def _bound(sc, pairs, pts, pend, cond, g_ref):
    """The per-(row, column) bound of the module docstring."""
    linv, w, terms, zd, kc = cond
    cpu = lambda t: None if t is None else t.detach().double().cpu()  # noqa: E731
    linv, w, terms, zd = cpu(linv), cpu(w), cpu(terms), cpu(zd)
    progs = kc.programs
    weights = [float(v) for v in kc.weights]
    P = 0 if pend is None else len(pend)
    Xl = torch.tensor(pts, dtype=torch.float64, requires_grad=True)
    mom = [oracle_moments(p.om, Xl, pend) for p in pairs]
    outs = []
    for mu, var, pe in mom:
        outs.append([mu, var] + ([] if pe is None else [pe[2][:, q] for q in range(P)]))
    grads = [[torch.autograd.grad(o.sum(), Xl, retain_graph=True)[0].abs() for o in os] for os in outs]

    def value_of(moms):
        # objective_value with the moments given: patch oracle_moments' results in through a small shim
        import tests.objective_grad_oracle as og

        it = iter(moms)
        saved = og.oracle_moments
        og.oracle_moments = lambda om, X, px: next(it)
        try:
            return objective_value([p.om for p in pairs], Xl.detach(), pend, linv, w, terms, zd, sc.cfg, progs,
                                   kc.scalarizer, weights)
        finally:
            og.oracle_moments = saved

    def partials(shift_mu, shift_var):
        moms, ins = [], []
        for (mu, var, pe), dm, dv in zip(mom, shift_mu, shift_var):
            m = (mu.detach() + dm).requires_grad_(True)
            v = (var.detach() + dv).clamp_min(rp.MIN_VARIANCE * 1e-6).requires_grad_(True)
            ins += [m, v]
            if pe is not None:
                c = pe[2].detach().clone().requires_grad_(True)
                ins.append(c)
                moms.append((m, v, (pe[0].detach(), pe[1].detach(), c)))
            else:
                moms.append((m, v, None))
        val = value_of(moms)
        if not val.requires_grad:  # the objective does not depend on the moments (a CONST program)
            return [[torch.zeros_like(m), torch.zeros_like(m)] + [torch.zeros_like(m)] * P for m, _, _ in moms]
        gs = torch.autograd.grad(val.sum(), ins, allow_unused=True)
        gs = [torch.zeros_like(t) if g is None else g for t, g in zip(ins, gs)]
        out, k = [], 0
        for pe in (x[2] for x in mom):
            o = [gs[k], gs[k + 1]]
            k += 2
            if pe is not None:
                o += [gs[k][:, q] for q in range(P)]
                k += 1
            out.append(o)
        return out

    M = len(pairs)
    A = partials([0.0] * M, [0.0] * M)
    tol = [posterior_tolerances(p.om, mom[m][0].detach()) for m, p in enumerate(pairs)]
    dA = [[torch.zeros_like(a) for a in Am] for Am in A]
    for sm in (-1.0, 1.0):
        for sv in (-1.0, 1.0):
            Ap = partials([sm * t[0] for t in tol], [sv * t[1] for t in tol])
            dA = [[torch.maximum(x, (a - b).abs()) for x, a, b in zip(dAm, Apm, Am)] for dAm, Apm, Am in zip(dA, Ap, A)]
    bound = 1e-3 * g_ref.abs() + 1e-7 * max(p.om.y_std for p in pairs)
    Pn_raw = None if pend is None else torch.tensor(pend, dtype=torch.float64)
    for m, p in enumerate(pairs):
        om = p.om
        sy, s2 = om.y_std, om.y_std**2
        Xn = rp._normalise(torch.tensor(pts, dtype=torch.float64), om.lo, om.rng)
        Pn = None if Pn_raw is None else rp._normalise(Pn_raw, om.lo, om.rng)
        beta = None if Pn is None else torch.cholesky_solve(rp.kernel_matrix(om.spec, om.Xn, Pn), om.L)
        T = [torch.zeros(len(pts), D, dtype=torch.float64) for _ in outs[m]]
        for r in range(len(pts)):
            xr = torch.tensor(pts[r], dtype=torch.float64)
            J = torch.autograd.functional.jacobian(
                lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), om.Xn)[0], xr).abs()
            k = rp.kernel_matrix(om.spec, Xn[r: r + 1], om.Xn)[0]
            u = torch.cholesky_solve(k[:, None], om.L)[:, 0]
            T[0][r] = sy * om.alpha.abs() @ J
            T[1][r] = 2 * s2 * u.abs() @ J
            if Pn is not None:
                JP = torch.autograd.functional.jacobian(
                    lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), Pn)[0], xr).abs()
                for q in range(P):
                    T[2 + q][r] = s2 * (JP[q] + beta[:, q].abs() @ J)
        eps32 = 2.0**-19 * math.sqrt(om.Xn.shape[0])
        for a, da, g, t in zip(A[m], dA[m], grads[m], T):
            bound = bound + eps32 * a.abs()[:, None] * t + da[:, None] * g
    # the value: the change the stated posterior tolerances can cause (first order, 1.5x), plus fp32 arithmetic
    vb = torch.zeros(len(pts), dtype=torch.float64)
    for Am, (dmu, dvar) in zip(A, tol):
        vb = vb + 1.5 * (Am[0].abs() * dmu + sum(a.abs() for a in Am[1:]) * dvar)
    return bound + _kink_allowance(sc, mom, progs, pend, linv, w, zd, g_ref), vb


def _kink_allowance(sc, mom, progs, pend, linv, w, zd, g_ref):
    if not sc.cfg.is_mc:
        return torch.zeros_like(g_ref)
    P = 0 if pend is None else len(pend)
    Q = P + 1
    n_kink = torch.zeros(g_ref.shape[0], dtype=torch.float64)
    for m, (mu, var, pe) in enumerate(mom):
        mu, var = mu.detach(), var.detach()
        zx = zd[:, m * Q + P]
        if P:
            c = pe[2].detach()
            r = c @ linv[m].T
            y = mu[None] + w[m] @ c.T + (var - (r * r).sum(-1)).clamp_min(0).sqrt()[None] * zx[:, None]
        else:
            y = mu[None] + var.sqrt()[None] * zx[:, None]
        for op, (a0, a1, a2) in progs[m]:
            for k in {"CLAMP": (a0, a1), "TWO_SIDED": (a2,)}.get(op, ()):
                if math.isfinite(k):
                    n_kink += ((y - k).abs() <= 1e-4 * (1 + abs(k))).sum(0).double()
    return (n_kink * 2.0 * g_ref.abs().amax(1) / zd.shape[0])[:, None].expand_as(g_ref)


def _check(sc, pairs, P, seed=0):
    pts, pend, z = _inputs(sc, P, seed)
    val, grad = sc.value_and_grad(torch.from_numpy(pts), pend, z)
    val2, grad2 = sc.value_and_grad(torch.from_numpy(pts), pend, z)
    assert torch.equal(val, val2) and torch.equal(grad, grad2)  # bit-identical repeated calls
    v_ref, g_ref, cond = _oracle(sc, pairs, pts, pend, z)
    bound, vdev = _bound(sc, pairs, pts, pend, cond, g_ref)
    err = (grad.double().cpu() - g_ref).abs()
    assert bool(torch.isfinite(grad).all())
    assert bool((err <= bound).all()), (float((err / bound).max()), float(err.max()))
    # the value: bb_objective_score's (the engine's own moments) within the stated per-row value bound
    scores = torch.as_tensor(sc.scores(pts, pend, seed, S))
    vb = 2e-4 + 1e-4 * v_ref.abs() + vdev
    assert bool(((val.double().cpu() - scores.double()).abs() <= vb).all()), (val, scores)
    return float((err / bound).max())


CASES = []
# every opcode (one target, NONE), qLogEI and qEI, with and without pending points
for name in PROGRAMS:
    for kind, P in (("qLogEI", 0), ("qEI", 8)):
        CASES.append((f"op-{name}-{kind}-P{P}", kind, "NONE", [name], "matern52", (24,), 1.3, P))
# scalarisers x MC kinds, two targets with different n (partial measurements)
for scal, progs in (("MEAN", ["bell", "clamp"]), ("GEOM_MEAN", ["bell", "sigmoid"])):
    for kind in MC:
        CASES.append((f"{scal}-{kind}", kind, scal, progs, "matern32", (20, 31), None, 1))
# analytic kinds: MEAN over affine targets, one minimised
for kind in ANALYTIC:
    CASES.append((f"analytic-{kind}", kind, "MEAN", ["affine", "minimised"], "rbf", (16, 40), 0.9, 0))
# families x output scale, M in {1, 2, 8}, n in {5, 64, 256}, P in {0, 1, 8, 31}
for i, fam in enumerate(FAMILIES):
    for os_ in (None, 1.6):
        M = (1, 2, 8, 2)[i]
        ns = tuple((5, 64, 256)[(i + m) % 3] for m in range(M))
        P = (0, 1, 8, 31)[(i + (os_ is None)) % 4]
        progs = (["bell", "pow", "add_mul", "sigmoid", "minimised", "clamp", "log_exp", "two_sided"])[:M]
        CASES.append((f"{fam}-os{os_}-M{M}", "qLogEI" if i % 2 == 0 else "qUCB", "NONE" if M == 1 else "GEOM_MEAN"
                      if i % 2 else "MEAN", progs, fam, ns, os_, P))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gradient_and_value_against_the_oracle(case):
    name, kind, scal, progs, fam, ns, os_, P = case
    pairs = [_Pair(fam, n, os_, seed=m) for m, n in enumerate(ns)]
    M = len(pairs)
    weights = [1.0] if M == 1 else list(np.linspace(1.0, 2.0, M) / np.linspace(1.0, 2.0, M).sum())
    if scal == "GEOM_MEAN":  # positive targets for the geometric mean
        progs = ["bell" if p in ("minimised", "log_exp", "two_sided", "pow", "clamp") else p for p in progs]
    sc = _scorer(pairs, kind, scal, [PROGRAMS[p] for p in progs], weights)
    worst = _check(sc, pairs, P)
    print(f"{name}: worst err/bound {worst:.3f}")


def test_continuous_2d_match_target_reaches_the_dense_grid_optimum():
    from baybe_b200.continuous import recommend_continuous_hybrid

    pair = _Pair("matern52", 14, None, seed=3)
    prog = [("BELL", (0.9, 0.3, 0.0))]
    sc = _scorer([pair], "qEI", "NONE", [prog], [1.0])
    disc = np.zeros((1, 0))
    # the inactive third column is held fixed
    pts, _, value = recommend_continuous_hybrid(sc, sc.cfg, disc, np.array([[0.0, 0.0, 0.5], [1.0, 1.0, 0.5]]), 1,
                                                seed=4, fixed={2: 0.5})
    g = np.stack(np.meshgrid(np.linspace(0, 1, 61), np.linspace(0, 1, 61)), -1).reshape(-1, 2)
    grid = np.concatenate([g, np.full((len(g), 1), 0.5)], 1)
    best = float(np.max(sc.scores(grid, None, 4, 512)))
    assert value >= best - 1e-4 * max(1.0, abs(best)), (value, best)


def test_hybrid_batch_reaches_an_exhaustive_greedy_search():
    from baybe_b200.continuous import recommend_continuous_hybrid

    pairs = [_Pair("matern52", 18, None, seed=1), _Pair("matern52", 12, None, seed=2)]
    sc = _scorer(pairs, "qEI", "GEOM_MEAN", [PROGRAMS["bell"], PROGRAMS["sigmoid"]], [0.5, 0.5])
    # 12 configurations over the first column, the second continuous, the third fixed
    disc = np.linspace(0, 1, 12)[:, None]
    cb = np.array([[0.0, 0.5], [1.0, 0.5]])
    pts, idx, value = recommend_continuous_hybrid(sc, sc.cfg, disc, cb, 3, seed=2, n_raw_samples=32, n_restarts=12,
                                                  fixed={1: 0.5}, n_samples=512)
    assert len(set(map(tuple, pts))) == 3
    # exhaustive greedy over the configurations x a dense grid of the continuous column
    grid = np.array([[c, t, 0.5] for c in disc[:, 0] for t in np.linspace(0, 1, 101)])
    chosen = []
    for _ in range(3):
        pend = np.array(chosen) if chosen else None
        v = sc.scores(grid, pend, 2, 512)
        chosen.append(grid[int(np.argmax(v))])
    want = sc.joint_value(np.array(chosen), None, 2, 512)
    assert value >= want - 2e-3 * max(1.0, abs(want)), (value, want)


def test_campaign_flows_on_the_engine():
    import sys

    from tests.test_continuous import REF, ROOT

    if REF is None:
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(REF)):
        if p not in sys.path:
            sys.path.append(p)
    from baybe_b200 import baybe_plugin
    from tests.test_continuous import _initial, _space
    from tests.test_objective_continuous import _campaign, _check_rows, _measure

    for kind in ("continuous", "hybrid"):
        for which in ("geom", "mean", "bell"):
            rng = np.random.default_rng(0)
            space = _space(kind, fixed=True)
            camp = _campaign(baybe_plugin, space, which)
            init = _measure(_initial(space, 6, rng), rng)
            if which == "geom":
                init.loc[init.index[:2], "purity"] = np.nan
            camp.add_measurements(init)
            q = 1 if which == "mean" else 3
            rec = camp.recommend(q)
            _check_rows(rec, space)
            camp.add_measurements(_measure(rec, rng))
            if which != "mean":
                rec2 = camp.recommend(3, pending_experiments=rec.iloc[:1])
                _check_rows(rec2, space)
                assert np.isfinite(camp.acquisition_values(rec2).to_numpy(dtype=float)).all()
                assert np.isfinite(camp.joint_acquisition_value(rec2))
