"""GPU tests of ``bb_hvi_grad`` (qEHVI / qLogEHVI on continuous and hybrid spaces): value and gradient against float64
autograd of the literal definition (tests/hvi_grad_oracle.py), the value against ``HviScorer.scores``
(``bb_hvi_score``), determinism, the optimiser against a dense grid and an exhaustive greedy search, Campaign flows on
the engine, and the models it does not serve.

Gradient bound, per row i and column j (tests/test_gpu_objective_continuous.py's bound):

    |g_ij - g_ref,ij| <= 1e-3 |g_ref,ij| + 1e-7 max_m s_y,m
        + sum_m EPS32_m * (|A_mu,m| T_mu,m + |A_var,m| T_var,m + sum_p |A_c,mp| T_c,mp)_j
        + sum_m sum over the partials A of max_corner |A(mu_m +- dmu_m, var_m +- dvar_m) - A| * |d moment / dx_j|
        + KINK_i,

with A_mu,m, A_var,m, A_c,mp the float64 partial derivatives of the value with respect to target m's moments, dmu /
dvar the stated posterior tolerances of tests/helpers.py, T the sums of absolute terms the device adds in fp32 and
EPS32 = 2^-19 sqrt(n_m).  KINK_i (qEHVI only: qLogEHVI's smoothed cell terms have a continuous derivative) allows for
the samples whose oriented y_m lies within 1e-4 (1 + |bound|) of a finite lower or upper cell bound: fp32 may put such a
sample on the other side, which moves the gradient by |jump| / S; the jump is taken as 2 max_j |g_ref,ij|, so
KINK_i = n_kink,i * 2 max_j |g_ref,ij| / S.  The value must agree with bb_hvi_score's within 2e-4 + 1e-4 |value| plus
1.5 times the first-order change the stated posterior tolerances can cause (the two compute the moments on different
fp32 paths).  With pending points that improve on the front, qLogEHVI's reported gradient is the kernel's times
sigmoid(v - log gain); the comparison is then against the oracle's gradient times the same factor at the oracle's value,
with the bound scaled by that factor plus |g_ref| sigmoid (1 - sigmoid) times the value bound."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import AcqConfig, DeviceGP, _lib
from baybe_b200.multiobjective import HviScorer, compute_ref_point
from oracle import reference_path as rp
from tests.continuous_oracle import oracle_moments
from tests.helpers import posterior_tolerances
from tests.hvi_grad_oracle import hvi_value, samples

pytestmark = pytest.mark.gpu

FAMILIES = ("matern12", "matern32", "matern52", "rbf")
S = 128
D = 3


class _Pair:
    """A device model and its oracle (``.om``, what the float64 stand-in reads)."""

    def __init__(self, family, n, outputscale, seed):
        rng = np.random.default_rng(seed)
        X = rng.uniform(0, 1, (n, D))
        sign = 1.0 if seed % 2 == 0 else -1.0
        y = sign * (np.sin(3 * X[:, 0]) + X[:, 1] ** 2) + 0.3 * seed + 0.05 * rng.normal(size=n)
        ls = np.array([0.45, 0.6, 0.0])  # one inactive column
        bounds = np.array([np.zeros(D), np.ones(D)])
        self.gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=bounds, family=family, lengthscale=ls,
                           noise=1e-2, outputscale=outputscale)
        spec = oracle.KernelSpec(family=family, lengthscale=ls[:2], active_dims=[0, 1], outputscale=outputscale)
        self.om = oracle.build_model(spec, X, y, bounds, noise=1e-2)
        self.X = X


def _scorer(pairs, kind):
    M = len(pairs)
    a = np.array([1.0, -1.0, 1.0, -1.0][:M])
    b = np.array([0.0, 2.0, 0.0, 2.0][:M])
    front = np.stack([oracle.posterior(p.om, pairs[0].X)[0].numpy() for p in pairs], 1) * a + b
    return HviScorer([p.gp for p in pairs], AcqConfig(kind=kind), a, b, compute_ref_point(front), front)


def _inputs(sc, P, seed=0):
    rng = np.random.default_rng(seed + 7)
    pts = rng.uniform(0.05, 0.95, (10, D))
    pend = rng.uniform(0, 1, (P, D)) if P else None
    return pts, pend, sc.base_samples(S, P, seed)


def _conditioning(sc, pend, z):
    """The step's constants as value_and_grad hands them to the kernel (host float64 linv / w, fp32 cells)."""
    P = 0 if pend is None else len(pend)
    zz = torch.as_tensor(z, dtype=torch.float64).reshape(-1, sc.M * (1 + P))
    if P == 0:
        linv = w = None
        decomps = sc._front_decomps
    else:
        _, linv_h, w_h, decomps, _ = sc._pending_parts(np.asarray(pend, dtype=np.float64), zz)
        linv = torch.from_numpy(linv_h).float().double()
        w = torch.from_numpy(w_h).float().double()
    lower, upper, counts = sc._device_cells(decomps)
    return linv, w, zz.float().double(), lower.double().cpu(), upper.double().cpu(), counts.cpu()


def _bound(sc, pairs, pts, pend, cond, g_ref):
    """The per-(row, column) bound and the value bound of the module docstring."""
    linv, w, zd, lower, upper, counts = cond
    log = sc.cfg.kind == "qLogEHVI"
    P = 0 if pend is None else len(pend)
    Xl = torch.tensor(pts, dtype=torch.float64, requires_grad=True)
    mom = [oracle_moments(p.om, Xl, pend) for p in pairs]
    outs = [[mu, var] + ([] if pe is None else [pe[2][:, q] for q in range(P)]) for mu, var, pe in mom]
    grads = [[torch.autograd.grad(o.sum(), Xl, retain_graph=True)[0].abs() for o in os] for os in outs]

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
        val = hvi_value(moms, linv, w, zd, lower, upper, counts, log, sc.a, sc.b, sc.cfg.tau_relu, sc.cfg.tau_max)
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
    vb = torch.zeros(len(pts), dtype=torch.float64)
    for Am, (dmu, dvar) in zip(A, tol):
        vb = vb + 1.5 * (Am[0].abs() * dmu + sum(a.abs() for a in Am[1:]) * dvar)
    if not log:  # KINK_i
        Y = samples([(mu.detach(), var.detach(), None if pe is None else (pe[0], pe[1], pe[2].detach()))
                     for mu, var, pe in mom], linv, w, zd, sc.a, sc.b)  # (S, B, M)
        n_kink = torch.zeros(len(pts), dtype=torch.float64)
        for s in range(Y.shape[0]):
            k = 0 if lower.shape[0] == 1 else s
            nc = int(counts[k])
            edges = torch.cat([lower[k, :nc], upper[k, :nc]], 0)  # (2C, M)
            near = ((Y[s][:, None, :] - edges[None]).abs() <= 1e-4 * (1 + edges.abs()[None])) & torch.isfinite(edges)
            n_kink += near.sum((1, 2)).double()
        bound = bound + (n_kink * 2.0 * g_ref.abs().amax(1) / Y.shape[0])[:, None]
    return bound, vb


def _check(sc, pairs, P, seed=0):
    pts, pend, z = _inputs(sc, P, seed)
    val, grad = sc.value_and_grad(torch.from_numpy(pts), pend, z)
    val2, grad2 = sc.value_and_grad(torch.from_numpy(pts), pend, z)
    assert torch.equal(val, val2) and torch.equal(grad, grad2)  # bit-identical repeated calls
    cond = _conditioning(sc, pend, z)
    px = None if pend is None else torch.tensor(pend, dtype=torch.float64)
    v_ref, g_ref = _oracle64(pairs, pts, px, cond, sc)
    bound, vdev = _bound(sc, pairs, pts, pend, cond, g_ref)
    # value_and_grad reports through the pending points' own improvement: qLogEHVI's reporter scales the gradient by
    # sigmoid(v - log gain), formed from the kernel's value, whose error is within the stated value bound
    gain = 0.0 if pend is None else sc._pending_parts(np.asarray(pend, dtype=np.float64),
                                                     torch.as_tensor(z, dtype=torch.float64))[4]
    if gain > 0.0 and sc.cfg.kind == "qLogEHVI":
        sig = torch.sigmoid(v_ref - math.log(gain))
        dv = 2e-4 + 1e-4 * v_ref.abs() + vdev
        bound = bound * sig[:, None] + (g_ref.abs() * (sig * (1 - sig) * dv)[:, None])
        g_ref = g_ref * sig[:, None]
    assert bool(torch.isfinite(grad).all())
    err = (grad - g_ref).abs()
    assert bool((err <= bound).all()), (float((err / bound).max()), float(err.max()))
    scores = torch.as_tensor(sc.scores(pts, pend, seed, S))
    vb = 2e-4 + 1e-4 * scores.abs() + vdev
    assert bool(((val - scores).abs() <= vb).all()), (val, scores)
    return float((err / bound).max())


def _oracle64(pairs, pts, px, cond, sc):
    """Float64 value and gradient of the definition (tests/hvi_grad_oracle.py) without the float32 rounding of the
    stand-in's outputs."""
    linv, w, zd, lower, upper, counts = cond
    X = torch.tensor(pts, dtype=torch.float64, requires_grad=True)
    moments = [oracle_moments(p.om, X, px) for p in pairs]
    val = hvi_value(moments, linv, w, zd, lower, upper, counts, sc.cfg.kind == "qLogEHVI", sc.a, sc.b,
                    sc.cfg.tau_relu, sc.cfg.tau_max)
    (g,) = torch.autograd.grad(val.sum(), X)
    return val.detach(), g


CASES = []
for fam in FAMILIES:
    for osc in (None, 1.7):
        CASES.append((f"{fam}-os{osc}-M2", fam, osc, (5, 64), "qEHVI", 0))
        CASES.append((f"{fam}-os{osc}-M2-log", fam, osc, (64, 5), "qLogEHVI", 1))
for M, ns in ((3, (5, 64, 256)), (4, (64, 5, 256, 64))):
    for kind in ("qEHVI", "qLogEHVI"):
        for P in (0, 1, 8, 31):
            CASES.append((f"M{M}-{kind}-P{P}", "matern52", 1.3, ns, kind, P))


@pytest.mark.parametrize("name, family, osc, ns, kind, P", CASES, ids=[c[0] for c in CASES])
def test_value_and_gradient_match_the_float64_oracle(name, family, osc, ns, kind, P):
    pairs = [_Pair(family, n, osc, seed=m) for m, n in enumerate(ns)]
    sc = _scorer(pairs, kind)
    _check(sc, pairs, P)


def test_continuous_optimum_and_hybrid_greedy_batch():
    """2-D: the optimum reaches the dense-grid optimum; hybrid (3 configurations x 1 continuous column, q = 2): every
    greedy step is at least as good as the configurations x a dense grid given the same pending points."""
    from baybe_b200.continuous import recommend_continuous_hybrid

    rng = np.random.default_rng(2)
    pairs = []
    for m in range(2):
        X = rng.uniform(0, 1, (12, 2))
        y = (np.sin(3 * X).sum(1)) * (1 if m == 0 else -1) + 0.3 * m
        pairs.append(DeviceGP(device="cuda", train_x=X, train_y=y, bounds=np.array([[0.0, 0.0], [1.0, 1.0]]),
                              family="matern52", lengthscale=np.full(2, 0.4), noise=1e-3, outputscale=1.2))
    a, b = np.array([1.0, -1.0]), np.array([0.0, 2.0])
    X0 = rng.uniform(0, 1, (8, 2))
    front = np.stack([gp.posterior(torch.from_numpy(X0).float().cuda())[0].double().cpu().numpy() for gp in pairs],
                     1) * a + b
    for kind in ("qEHVI", "qLogEHVI"):
        sc = HviScorer(pairs, AcqConfig(kind=kind), a, b, compute_ref_point(front), front)
        g = np.linspace(0, 1, 101)
        grid = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
        best = float(sc.scores(grid, None, 4, 128).max())
        _, _, value = recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), np.array([[0.0, 0.0], [1.0, 1.0]]),
                                                  1, n_samples=128, seed=4, n_raw_samples=64, n_restarts=8)
        assert value >= best - 1e-4 * max(1.0, abs(best)), (kind, value, best)
        disc = np.array([[0.1], [0.5], [0.9]])
        pts, idx, _ = recommend_continuous_hybrid(sc, sc.cfg, disc, np.array([[0.0], [1.0]]), 2, n_samples=128,
                                                  seed=6, n_raw_samples=32, n_restarts=8)
        gg = np.linspace(0, 1, 401)
        cand = np.concatenate([np.repeat(disc, len(gg), 0), np.tile(gg, 3)[:, None]], 1)
        for step in range(2):
            pend = pts[:step] if step else None
            best = float(sc.scores(cand, pend, 6, 128).max())
            got = float(sc.scores(pts[step: step + 1], pend, 6, 128)[0])
            assert got >= best - 1e-4 * max(1.0, abs(best)), (kind, step, got, best)


@pytest.fixture()
def bb():
    import sys

    from tests.test_continuous import REF, ROOT

    if REF is None:
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(REF)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe_b200 import baybe_plugin

    return baybe_plugin


@pytest.mark.parametrize("acq", ["qEHVI", "qLogEHVI"])
@pytest.mark.parametrize("kind", ["continuous", "hybrid"])
def test_campaign_flow_on_the_engine(bb, kind, acq):
    from tests.test_hvi_continuous import campaign_flow

    campaign_flow(bb, kind, acq)


def test_wide_and_task_models_are_unsupported():
    """Both are rejected by the host checks, before any device access."""
    from tests.test_gpu_wide import WIDE

    w = WIDE["d100_n200_m52"]()
    wide = DeviceGP(device="cuda", **w.gp_kwargs())
    assert wide.model.wide == 1
    small = _Pair("matern52", 12, None, seed=0).gp
    for gp, msg in ((wide, "wide-feature"), (small, "task parameter")):
        sc = HviScorer([gp, gp], AcqConfig(kind="qEHVI"), [1.0, 1.0], [0.0, 0.0], [-10.0, -10.0], np.zeros((1, 2)))
        x = torch.zeros((4, gp.d), dtype=torch.float32)
        saved = gp.model.task_col
        if gp is small:
            gp.model.task_col = 0  # flagged as a task model: the check fires on the host
        try:
            with pytest.raises(Exception, match=msg):
                sc.value_and_grad(x, None, sc.base_samples(32, 0, 1))
        finally:
            gp.model.task_col = saved
