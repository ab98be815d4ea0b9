"""GPU tests of ``bb_objective_grad_large``, the gradient path of desirability objectives and transformed targets for
models with n_pad > 256 or wide features: value and gradient against float64 autograd of the literal definition
(tests/objective_grad_oracle.py), values against ``ObjectiveScorer.scores`` (``bb_objective_score``), agreement with
``bb_objective_grad`` where both apply, determinism, the shared-memory limit, the optimiser's quality and Campaign
flows on the engine.

Gradient bound: test_gpu_objective_continuous.py's per-element bound, summed over the targets, with EPS32_m =
2^-19 sqrt(n_m) for target m (test_gpu_acq_grad_large.py explains the growth in n); the kernel rows' Jacobians are
formed in forward mode.  For qEI the kink of max(o - best_f, 0) gets the allowance test_gpu_objective_continuous.py's
docstring describes, per sample within roundoff of it (``_best_f_kink_allowance``).  Values: within 2e-4 + 1e-4 |v|
plus 1.5 times the first-order change the stated posterior tolerances can cause, those tolerances grown by sqrt(n_m / 256) past n_m = 256, of the oracle's value, and within
twice that of bb_objective_score's.  The scoring path has no Matern-1/2 on wide models, so there the value is compared
with the oracle only."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import DeviceGP
from baybe_b200 import objectives as ob
from baybe_b200.engine import objective_grad_op
from baybe_b200.objectives import CompiledObjective, ObjectiveScorer, evaluate_objective
from oracle import reference_path as rp
from tests.continuous_oracle import oracle_moments
from tests.helpers import posterior_tolerances
from tests.objective_grad_oracle import objective_grad_f64, objective_value
from tests.test_gpu_objective_continuous import ANALYTIC, MC, PROGRAMS, _kink_allowance

pytestmark = pytest.mark.gpu

S = 128


class _Pair:
    """A device model on d columns (column 1 inactive for d > 1) and its oracle."""

    def __init__(self, family, n, d, outputscale, seed):
        rng = np.random.default_rng(seed)
        X = rng.uniform(0, 1, (n, d))
        y = np.sin(3 * X[:, 0]) + X[:, min(2, d - 1)] ** 2 + 0.3 * seed + 0.05 * rng.normal(size=n)
        ls = np.full(d, 0.45 * math.sqrt(d))
        if d > 1:
            ls[1] = 0.0
        active = [j for j in range(d) if ls[j] > 0]
        bounds = np.array([np.zeros(d), np.ones(d)])
        self.gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=bounds, family=family, lengthscale=ls,
                           noise=1e-2, outputscale=outputscale)
        spec = oracle.KernelSpec(family=family, lengthscale=ls[active], active_dims=active, outputscale=outputscale)
        self.om = oracle.build_model(spec, X, y, bounds, noise=1e-2)
        self.X, self.d, self.family = X, d, family


def _scorer(pairs, kind, scal, progs, weights, beta=0.6):
    comp = CompiledObjective([f"t{m}" for m in range(len(pairs))], progs, scal, weights)
    analytic = None if kind in MC else comp
    from baybe_b200 import AcqConfig

    sc = ObjectiveScorer([p.gp for p in pairs], AcqConfig(kind, best_f=0.0, beta=beta), comp, analytic)
    means = np.stack([oracle.posterior(p.om, pairs[0].X)[0].numpy() for p in pairs], 1)
    sc.cfg = AcqConfig(kind, best_f=float(np.max(evaluate_objective(comp, means))), beta=beta)
    return sc


def _large(pairs):
    return objective_grad_op([p.gp.model for p in pairs]) is torch.ops.baybe_b200.objective_grad_large


def _inputs(sc, pairs, P, seed, on_rows):
    d = pairs[0].d
    rng = np.random.default_rng(seed + 7)
    X0 = pairs[0].X
    near = (X0[:3] + 1e-2 * rng.normal(size=(3, d))).clip(0, 1)
    pts = np.vstack([rng.uniform(0.05, 0.95, (7, d)), near] + ([X0[3:5]] if on_rows else []))
    pend = rng.uniform(0, 1, (P, d)) if P else None
    z = sc.base_samples(S, P, seed) if sc.cfg.is_mc else None
    return pts, pend, z


def _oracle(sc, pairs, pts, pend, z):
    from baybe_b200 import _lib

    P, stats, linv, w, terms, zd = sc.conditioning(pend, z)
    kc = sc.kernel_comp
    ops, args, n_ops = kc.flat()
    a = (pts, pend, None, linv, w, terms, zd, _lib.ACQ_KIND[sc.cfg.kind], sc.cfg.params(),
         _lib.OBJ_SCALARIZER[kc.scalarizer], ops, args, n_ops, [float(v) for v in kc.weights])
    val, g = objective_grad_f64(pairs, *a)
    return val.double(), g.double(), (linv, w, terms, zd, kc)


def _bound(sc, pairs, pts, pend, cond, g_ref):
    """The per-(row, column) gradient bound and the value bound of the module docstring."""
    linv, w, terms, zd, kc = cond
    cpu = lambda t: None if t is None else t.detach().double().cpu()  # noqa: E731
    linv, w, terms, zd = cpu(linv), cpu(w), cpu(terms), cpu(zd)
    progs, weights = kc.programs, [float(v) for v in kc.weights]
    P = 0 if pend is None else len(pend)
    d = pts.shape[1]
    Xl = torch.tensor(pts, dtype=torch.float64, requires_grad=True)
    mom = [oracle_moments(p.om, Xl, pend) for p in pairs]
    outs = [[mu, var] + ([] if pe is None else [pe[2][:, q] for q in range(P)]) for mu, var, pe in mom]
    grads = [[torch.autograd.grad(o.sum(), Xl, retain_graph=True)[0].abs() for o in os] for os in outs]

    def value_of(moms):
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
        if not val.requires_grad:  # a CONST program everywhere
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
        T = [torch.zeros(len(pts), d, dtype=torch.float64) for _ in outs[m]]
        for r in range(len(pts)):
            xr = torch.tensor(pts[r], dtype=torch.float64)
            J = torch.autograd.functional.jacobian(
                lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), om.Xn)[0], xr,
                vectorize=True, strategy="forward-mode").abs()
            k = rp.kernel_matrix(om.spec, Xn[r: r + 1], om.Xn)[0]
            u = torch.cholesky_solve(k[:, None], om.L)[:, 0]
            T[0][r] = sy * om.alpha.abs() @ J
            T[1][r] = 2 * s2 * u.abs() @ J
            if Pn is not None:
                JP = torch.autograd.functional.jacobian(
                    lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), Pn)[0], xr,
                    vectorize=True, strategy="forward-mode").abs()
                for q in range(P):
                    T[2 + q][r] = s2 * (JP[q] + beta[:, q].abs() @ J)
        eps32 = 2.0**-19 * math.sqrt(om.Xn.shape[0])
        for a, da, g, t in zip(A[m], dA[m], grads[m], T):
            bound = bound + eps32 * a.abs()[:, None] * t + da[:, None] * g
    vb = torch.zeros(len(pts), dtype=torch.float64)
    for Am, (dmu, dvar), p in zip(A, tol, pairs):
        grow = math.sqrt(max(1.0, p.om.Xn.shape[0] / 256))
        vb = vb + 1.5 * grow * (Am[0].abs() * dmu + sum(a.abs() for a in Am[1:]) * dvar)
    return bound + _kink_allowance(sc, mom, progs, pend, linv, w, zd, g_ref), vb


def _best_f_kink_allowance(sc, pairs, pts, pend, cond):
    """qEI: a sample whose objective o lies within 1e-4 (1 + |best_f|) of best_f, the kink of max(o - best_f, 0), may
    fall on the other side of it in fp32, which moves the gradient by its share of the join (at most 1) times
    |do_s/dx| / S.  Each such sample adds 2 |do_s/dx| / S, with do_s/dx from float64 autograd of the oracle's sample."""
    from tests.objective_oracle import objective

    allow = torch.zeros(pts.shape, dtype=torch.float64)
    if sc.cfg.kind != "qEI":
        return allow
    linv, w, _, zd, kc = cond
    P = 0 if pend is None else len(pend)
    Q = P + 1
    X = torch.tensor(pts, dtype=torch.float64, requires_grad=True)
    px = None if pend is None else torch.as_tensor(pend, dtype=torch.float64)
    zd = torch.as_tensor(zd).detach().double().cpu()
    ys = []
    for m, p in enumerate(pairs):
        mu, var, pe = oracle_moments(p.om, X, px)
        zx = zd[:, m * Q + P]
        if P == 0:
            ys.append(mu[None] + var.clamp_min(0).sqrt()[None] * zx[:, None])
            continue
        c = pe[2]
        r = c @ torch.as_tensor(linv[m]).detach().double().cpu().T
        sd = (var - (r * r).sum(-1)).clamp_min(0).sqrt()
        ys.append(mu[None] + torch.as_tensor(w[m]).detach().double().cpu() @ c.T + sd[None] * zx[:, None])
    o = objective(kc.programs, kc.scalarizer, [float(v) for v in kc.weights], torch.stack(ys, -1))  # (S, B)
    if not o.requires_grad:  # a CONST program: no sample moves with x
        return allow
    bf = sc.cfg.best_f
    for s, i in ((o.detach() - bf).abs() <= 1e-4 * (1 + abs(bf))).nonzero().tolist():
        (g,) = torch.autograd.grad(o[s, i], X, retain_graph=True)
        allow[i] += 2 * g[i].abs() / o.shape[0]
    return allow


def _check(sc, pairs, P, seed=0, on_rows=True):
    """Repeats bit-identical; gradient within the bound of the oracle's; the value within the value bound of the
    oracle's and twice that of bb_objective_score's.  Returns the worst gradient err / bound."""
    pts, pend, z = _inputs(sc, pairs, P, seed, on_rows)
    val, grad = sc.value_and_grad(torch.from_numpy(pts), pend, z)
    val2, grad2 = sc.value_and_grad(torch.from_numpy(pts), pend, z)
    assert torch.equal(val, val2) and torch.equal(grad, grad2)
    v_ref, g_ref, cond = _oracle(sc, pairs, pts, pend, z)
    bound, vdev = _bound(sc, pairs, pts, pend, cond, g_ref)
    bound = bound + _best_f_kink_allowance(sc, pairs, pts, pend, cond)
    err = (grad.double().cpu() - g_ref).abs()
    assert bool(torch.isfinite(grad).all())
    worst = int((err / bound).argmax())
    assert bool((err <= bound).all()), (float((err / bound).max()), float(err.max()), divmod(worst, err.shape[1]),
                                        float(grad.flatten()[worst]), float(g_ref.flatten()[worst]))
    vb = 2e-4 + 1e-4 * v_ref.abs() + vdev
    assert bool(((val.double().cpu() - v_ref).abs() <= vb).all()), (val, v_ref)
    if not (pairs[0].family == "matern12" and any(p.gp.model.wide for p in pairs)):
        scores = torch.as_tensor(sc.scores(pts, pend, seed, S)).double()
        assert bool(((val.double().cpu() - scores).abs() <= 2 * vb).all()), (val, scores)
    return float((err / bound).max())


_GEOM = ["bell", "sigmoid", "bell", "sigmoid", "bell", "sigmoid", "bell", "sigmoid"]
_ALL8 = ["bell", "pow", "add_mul", "sigmoid", "minimised", "clamp", "log_exp", "two_sided"]
# (name, kind, scalarizer, programs, family, n per target, d, outputscale, P)
CASES = [
    ("qLogEI-geom-m52", "qLogEI", "GEOM_MEAN", ["bell", "sigmoid"], "matern52", (320, 257), 4, 1.3, 0),
    ("qLogEI-none-rbf-n1000", "qLogEI", "NONE", ["add_mul"], "rbf", (1000,), 1, None, 8),
    ("qEI-mean-m32", "qEI", "MEAN", ["bell", "clamp"], "matern32", (512, 300), 4, None, 8),
    ("qEI-none-const", "qEI", "NONE", ["const"], "matern52", (320,), 4, None, 0),
    ("qUCB-mixed-200-700", "qUCB", "GEOM_MEAN", ["bell", "sigmoid"], "rbf", (200, 700), 4, 1.6, 1),
    ("qSR-m12-M3", "qSR", "MEAN", ["two_sided", "pow", "log_exp"], "matern12", (320, 257, 400), 4, None, 0),
    ("qPI-M8-d20-P31", "qPI", "MEAN", _ALL8, "matern52", (257, 320, 512, 1000, 300, 400, 600, 260), 20, None, 31),
    ("qLogEI-M8-geom", "qLogEI", "GEOM_MEAN", _GEOM, "matern32", (300,) * 8, 4, 1.2, 0),
    ("qEI-mixed-100-300", "qEI", "GEOM_MEAN", ["bell", "sigmoid"], "matern32", (100, 300), 4, None, 8),
    ("qLogEI-none-affine", "qLogEI", "NONE", ["affine"], "matern12", (512,), 20, 1.4, 1),
] + [(f"analytic-{k}", k, "MEAN", ["affine", "minimised"], fam, (300, 700), 4, 0.9, 0)
     for k, fam in zip(ANALYTIC, ("rbf", "matern32", "matern52", "matern12", "rbf", "matern52"))]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gradient_and_value_against_the_oracle(case):
    name, kind, scal, progs, fam, ns, d, os_, P = case
    pairs = [_Pair(fam, n, d, os_, seed=m) for m, n in enumerate(ns)]
    assert _large(pairs)
    M = len(pairs)
    weights = [1.0] if M == 1 else list(np.linspace(1.0, 2.0, M) / np.linspace(1.0, 2.0, M).sum())
    sc = _scorer(pairs, kind, scal, [PROGRAMS[p] for p in progs], weights)
    worst = _check(sc, pairs, P, on_rows=fam != "matern12")  # Matern-1/2 has a kink at distance 0
    print(f"{name}: worst err/bound {worst:.3f}")


def _wide_pairs(family="matern52"):
    """Two targets on one d = 100, n = 200 design: each model wide by d (n_pad 256 x d_pad 100 x 4 B > 56 KB)."""
    out = []
    rng = np.random.default_rng(21)
    X = rng.uniform(0, 1, (200, 100))
    ls = np.linspace(1.5, 4.0, 100)
    bounds = np.array([np.zeros(100), np.ones(100)])
    for m in range(2):
        y = np.sin(3 * X[:, m]) + X[:, 50 + m] ** 2 + 0.05 * rng.normal(size=200)
        p = _Pair.__new__(_Pair)
        p.gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=bounds, family=family, lengthscale=ls, noise=1e-2)
        spec = oracle.KernelSpec(family=family, lengthscale=ls, active_dims=list(range(100)))
        p.om = oracle.build_model(spec, X, y, bounds, noise=1e-2)
        p.X, p.d, p.family = X, 100, family
        assert p.gp.model.wide == 1
        out.append(p)
    return out


@pytest.mark.parametrize("kind, P", [("qLogEI", 0), ("qEI", 8), ("qUCB", 1), ("EI", 0)])
def test_two_target_wide_by_d_model(kind, P):
    pairs = _wide_pairs()
    assert _large(pairs)
    scal, progs = ("MEAN", ["affine", "minimised"]) if kind == "EI" else ("GEOM_MEAN", ["bell", "sigmoid"])
    sc = _scorer(pairs, kind, scal, [PROGRAMS[p] for p in progs], [0.5, 0.5])
    print(f"d100_n200 wide {kind} P={P}: worst err/bound {_check(sc, pairs, P):.3f}")


def test_matern12_wide_model_against_the_oracle_only():
    pairs = _wide_pairs("matern12")
    sc = _scorer(pairs, "qLogEI", "GEOM_MEAN", [PROGRAMS["bell"], PROGRAMS["sigmoid"]], [0.5, 0.5])
    print(f"d100_n200 wide matern12: worst err/bound {_check(sc, pairs, 0, on_rows=False):.3f}")


# ---- agreement with bb_objective_grad where both apply ---------------------------------------------------------------
@pytest.mark.parametrize("shape", [((5, 64), 1, 0, "qLogEI"), ((64, 256), 4, 8, "qEI"), ((200, 256, 31), 20, 31, "qUCB"),
                                   ((40, 100), 4, 0, "EI")],
                         ids=["d1-p0", "d4-p8", "d20-p31-M3", "d4-analytic"])
@pytest.mark.parametrize("family", ("matern12", "matern32", "matern52", "rbf"))
def test_agrees_with_bb_objective_grad_on_shared_shapes(family, shape):
    """With d < 32 and n_pad <= 256 both kernels form every target's moments in the same order and take the value and
    its partials from the same device function (objective_point_partials), so the values are bit-identical; the
    gradients differ in the order of the reverse pass's sums and are held to the bound around each other."""
    ns, d, P, kind = shape
    pairs = [_Pair(family, n, d, 1.3, seed=m + 3) for m, n in enumerate(ns)]
    assert not _large(pairs)
    M = len(pairs)
    if kind == "EI":
        scal, progs = "MEAN", ["affine", "minimised"]
    else:
        scal, progs = ("GEOM_MEAN", (["bell", "sigmoid", "bell"])[:M]) if M > 1 else ("NONE", ["add_mul"])
    sc = _scorer(pairs, kind, scal, [PROGRAMS[p] for p in progs], [1.0 / M] * M)
    pts, pend, z = _inputs(sc, pairs, P, 5, on_rows=False)
    xd = pairs[0].gp.prepare(torch.from_numpy(pts)).to(torch.float32).contiguous()
    seen = {}

    def spy(op):
        def call(*a):
            seen["args"] = a
            return op(*a)
        return call

    # capture the arguments the seam passes, then call both ops on them
    orig = ob.objective_grad_op
    ob.objective_grad_op = lambda models: spy(orig(models))
    try:
        sc.value_and_grad(torch.from_numpy(pts), pend, z)
    finally:
        ob.objective_grad_op = orig
    args = seen["args"]
    assert torch.equal(args[0], xd)
    v0, g0 = torch.ops.baybe_b200.objective_grad(*args)
    v1, g1 = torch.ops.baybe_b200.objective_grad_large(*args)
    assert torch.equal(v0, v1), (v0, v1)
    v_ref, g_ref, cond = _oracle(sc, pairs, pts, pend, z)
    bound, _ = _bound(sc, pairs, pts, pend, cond, g_ref)
    assert bool(((g1.double().cpu() - g0.double().cpu()).abs() <= bound).all())


def test_repeated_calls_at_10k_points_with_8_pending_are_bit_identical():
    pairs = [_Pair("matern52", n, 4, None, seed=m) for m, n in enumerate((700, 300))]
    sc = _scorer(pairs, "qLogEI", "GEOM_MEAN", [PROGRAMS["bell"], PROGRAMS["sigmoid"]], [0.5, 0.5])
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.uniform(0, 1, (10_000, 4)))
    pend = rng.uniform(0, 1, (8, 4))
    z = sc.base_samples(512, 8, 3)
    v0, g0 = sc.value_and_grad(x, pend, z)
    v1, g1 = sc.value_and_grad(x, pend, z)
    assert torch.equal(v0, v1) and torch.equal(g0, g1)
    assert bool(torch.isfinite(v0).all() and torch.isfinite(g0).all())


def test_shared_memory_overflow_names_the_sizes():
    """Eight targets on one n = 1000, d = 4000 model: a [8][4000], the slopes and L^-1 k [8][1024] and the base samples
    [1024][8] need more than 227 KB."""
    from baybe_b200 import AcqConfig, _lib

    rng = np.random.default_rng(0)
    X = rng.uniform(0, 1, (1000, 4000))
    gp = DeviceGP(device="cuda", train_x=X, train_y=X[:, 0], bounds=np.array([np.zeros(4000), np.ones(4000)]),
                  family="matern52", lengthscale=np.full(4000, 20.0), noise=1e-2)
    M = 8
    comp = CompiledObjective([f"t{m}" for m in range(M)], [PROGRAMS["bell"]] * M, "GEOM_MEAN", [1.0 / M] * M)
    ops, args, n_ops = comp.flat()
    x = torch.rand(4, 4000, device="cuda")
    z = torch.randn(1024, M, device="cuda")
    assert gp.model.n_pad == 1024
    with pytest.raises(NotImplementedError, match=r"M=8 targets with n_pad up to 1024 .*d_pad=\d+ and P=0 need \d+ bytes"):
        torch.ops.baybe_b200.objective_grad_large(x, [gp.handle] * M, None, [], None, None, None, z,
                                                  _lib.ACQ_KIND["qLogEI"], AcqConfig("qLogEI", best_f=0.0).params(),
                                                  _lib.OBJ_SCALARIZER["GEOM_MEAN"], ops, args, n_ops, [1.0 / M] * M)


# ---- optimiser quality ---------------------------------------------------------------------------------------------
def test_continuous_2d_match_target_reaches_the_dense_grid_optimum_at_n300():
    from baybe_b200.continuous import recommend_continuous_hybrid

    pair = _Pair("matern52", 300, 3, None, seed=3)
    assert _large([pair])
    sc = _scorer([pair], "qEI", "NONE", [[("BELL", (0.9, 0.3, 0.0))]], [1.0])
    pts, _, value = recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)),
                                                np.array([[0.0, 0.0, 0.5], [1.0, 1.0, 0.5]]), 1, seed=4,
                                                fixed={2: 0.5})
    g = np.stack(np.meshgrid(np.linspace(0, 1, 61), np.linspace(0, 1, 61)), -1).reshape(-1, 2)
    grid = np.concatenate([g, np.full((len(g), 1), 0.5)], 1)
    best = float(np.max(sc.scores(grid, None, 4, 512)))
    assert value >= best - 1e-4 * max(1.0, abs(best)), (value, best)


def test_hybrid_batch_at_n300_reaches_an_exhaustive_greedy_search():
    from baybe_b200.continuous import recommend_continuous_hybrid

    pairs = [_Pair("matern52", 300, 3, None, seed=1), _Pair("matern52", 180, 3, None, seed=2)]
    assert _large(pairs)
    sc = _scorer(pairs, "qEI", "GEOM_MEAN", [PROGRAMS["bell"], PROGRAMS["sigmoid"]], [0.5, 0.5])
    disc = np.linspace(0, 1, 12)[:, None]
    cb = np.array([[0.0, 0.5], [1.0, 0.5]])
    pts, idx, value = recommend_continuous_hybrid(sc, sc.cfg, disc, cb, 3, seed=2, n_raw_samples=32, n_restarts=12,
                                                  fixed={1: 0.5}, n_samples=512)
    assert len(set(map(tuple, pts))) == 3
    grid = np.array([[c, t, 0.5] for c in disc[:, 0] for t in np.linspace(0, 1, 101)])
    chosen = []
    for _ in range(3):
        pend = np.array(chosen) if chosen else None
        v = sc.scores(grid, pend, 2, 512)
        chosen.append(grid[int(np.argmax(v))])
    want = sc.joint_value(np.array(chosen), None, 2, 512)
    assert value >= want - 2e-3 * max(1.0, abs(want)), (value, want)


# ---- Campaign flows on the CUDA engine -----------------------------------------------------------------------------
@pytest.fixture()
def flows(monkeypatch):
    import sys

    from tests import test_continuous as tc

    if tc.REF is None:
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(tc.ROOT / "tests" / "shims"), str(tc.REF)):
        if p not in sys.path:
            sys.path.append(p)
    picked = []
    orig = ob.objective_grad_op

    def spy(models):
        op = orig(models)
        picked.append(op)
        return op

    monkeypatch.setattr(ob, "objective_grad_op", spy)
    return tc, picked


def _geom_campaign(space):
    from baybe_b200 import baybe_plugin
    from tests.test_objective_continuous import _campaign

    return _campaign(baybe_plugin, space, "geom")


@pytest.mark.parametrize("partial", (False, True), ids=["full", "partial-300-150"])
def test_continuous_desirability_campaign_with_300_measurements(flows, partial):
    tc, picked = flows
    from tests.test_objective_continuous import _check_rows, _measure

    rng = np.random.default_rng(3)
    space = tc._space("continuous", fixed=True)
    camp = _geom_campaign(space)
    init = _measure(tc._initial(space, 300, rng), rng)
    if partial:  # the purity model gets 150 rows, the yield model 300
        init.loc[init.index[:150], "purity"] = np.nan
    camp.add_measurements(init)
    for q in (1, 3):
        rec = camp.recommend(q)
        assert len(rec) == q
        _check_rows(rec, space)
    assert torch.ops.baybe_b200.objective_grad_large in picked
    vals = camp.acquisition_values(rec)
    assert len(vals) == 3 and np.all(np.isfinite(vals.to_numpy(dtype=float)))
    assert np.isfinite(camp.joint_acquisition_value(rec))


def test_hybrid_match_triangular_campaign_on_a_model_wide_by_d(flows):
    tc, picked = flows
    from baybe import Campaign
    from baybe.objectives import SingleTargetObjective
    from baybe.parameters import CategoricalParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget

    from baybe_b200 import baybe_plugin
    from baybe_b200.surrogates import GaussianProcessSurrogate

    rng = np.random.default_rng(7)
    base = tc._space("continuous")
    space = SearchSpace.from_product([CategoricalParameter("substance", values=[f"s{i}" for i in range(100)],
                                                           encoding="OHE")] + list(base.continuous.parameters))
    d = len(space.comp_rep_columns)
    assert d == 102
    rec_ = baybe_plugin.B200BotorchRecommender(
        surrogate_model=GaussianProcessSurrogate(hyperparameters={"lengthscale": np.full(d, 0.5), "noise": 1e-3,
                                                                  "mean_const": 0.0}),
        n_mc_samples=64, n_raw_samples=16, n_restarts=3)
    camp = Campaign(space, SingleTargetObjective(NumericalTarget.match_triangular("yield", 1.5, width=2.0)), rec_)
    camp.add_measurements(tc._measure(tc._initial(space, 140, rng), rng))
    rec = camp.recommend(2)
    assert len(rec) == 2 and rec["substance"].isin([f"s{i}" for i in range(100)]).all()
    assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
    assert torch.ops.baybe_b200.objective_grad_large in picked
    assert np.all(np.isfinite(camp.acquisition_values(rec).to_numpy(dtype=float)))
