"""GPU tests of the gradient path: ``bb_acq_grad`` against float64 autograd of the oracle (tests/continuous_oracle.py),
its values against ``gp.score`` / ``gp.score_joint``, determinism, and the quality of the continuous and hybrid
optimiser (baybe_b200/continuous.py) against dense oracle searches.

Gradient bound, per row i and column j, with no outlier allowance:

    |g_ij - g_ref,ij| <= 1e-3 |g_ref,ij| + EPS32 * (|A_mu| T_mu + |A_var| T_var + sum_p |A_c,p| T_c,p)_j
                         + sum over the partials A of max_corner |A(mu +- dmu, var +- dvar) - A| * |d moment / dx_j|
                         + 1e-7 * s_y,

where A_mu, A_var, A_c are the float64 partial derivatives of the value with respect to the moments, dmu / dvar the
stated posterior tolerances of tests/helpers.py, and T the sums of absolute terms the device adds in fp32:
T_mu = s_y sum_i |alpha_i| |dk_i/dx|, T_var = 2 s_y^2 sum_i |u_i| |dk_i/dx| (u = K~^-1 k), T_c,p = s_y^2 (|dk(x, x_p)/dx| +
sum_i |beta_p,i| |dk_i/dx|).  EPS32 = 2^-19 sqrt(n) is 32 units of fp32 roundoff of such a sum (the kernel values themselves carry a few
units from the rounded scaled rows).  Near training rows
sigma^2 and its gradient cancel in fp32: T_var carries that cancellation, the moment corners carry the resulting
change of the partials."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import AcqConfig, DeviceGP, sobol_normal_samples
from baybe_b200._lib import GRAD_KINDS
from oracle import reference_path as rp
from tests.continuous_oracle import acq_of_moments, oracle_moments, oracle_value_and_grad
from tests.helpers import posterior_tolerances, score_bounds

pytestmark = pytest.mark.gpu

FAMILIES = ("matern12", "matern32", "matern52", "rbf")
MC = ("qLogEI", "qEI", "qUCB", "qSR", "qPI")
S = 128


def _setup(family, d, n, outputscale, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (n, d))
    y = np.sin(4 * X[:, : min(d, 3)]).sum(1) + 0.05 * rng.normal(size=n)
    ls = np.full(d, 0.35 * math.sqrt(max(d, 1)))
    if d > 1:
        ls[1] = 0.0  # an inactive column
    bounds = np.array([np.zeros(d), np.ones(d)])
    kw = dict(train_x=X, train_y=y, bounds=bounds, family=family, lengthscale=ls, noise=1e-2, outputscale=outputscale)
    gp = DeviceGP(device="cuda", **kw)
    active = [j for j in range(d) if ls[j] > 0]
    spec = oracle.KernelSpec(family=family, lengthscale=ls[active], active_dims=active, outputscale=outputscale)
    om = oracle.build_model(spec, X, y, bounds, noise=1e-2)
    near = min(6, n)
    pts = np.vstack([rng.uniform(0, 1, (12, d)), X[:near] + 1e-2 * rng.normal(size=(near, d))]).clip(0, 1)
    return gp, om, X, pts


def _acq(kind, om, X):
    spec = oracle.AcqSpec(kind, beta=0.7)
    spec.best_f = oracle.best_f_from_training(om, X, spec)
    return spec, AcqConfig(kind, best_f=spec.best_f, beta=0.7)


def _bound(om, spec, pts, z, pend, g_ref):
    """The per-(row, column) bound of the module docstring."""
    Xl = torch.tensor(pts, dtype=torch.float64, requires_grad=True)
    mu, var, pe = oracle_moments(om, Xl, pend)
    d = pts.shape[1]
    grads = []
    outs = [mu, var] + ([] if pe is None else [pe[2][:, q] for q in range(pe[2].shape[1])])
    for o in outs:
        (gx,) = torch.autograd.grad(o.sum(), Xl, retain_graph=True)
        grads.append(gx.abs())

    def partials(m, v, c):
        m = m.detach().clone().requires_grad_(True)
        v = v.detach().clone().requires_grad_(True)
        ins = [m, v]
        pp = None
        if pe is not None:
            c = c.detach().clone().requires_grad_(True)
            ins.append(c)
            pp = (pe[0].detach(), pe[1].detach(), c)
        val = acq_of_moments(spec, m, v, pp, z)
        gs = torch.autograd.grad(val.sum(), ins, allow_unused=True)
        gs = [torch.zeros_like(t) if g is None else g for t, g in zip(ins, gs)]
        return [gs[0], gs[1]] + ([] if pe is None else [gs[2][:, q] for q in range(gs[2].shape[1])])

    c0 = None if pe is None else pe[2]
    A = partials(mu, var, c0)
    dmu, dvar = posterior_tolerances(om, mu.detach())
    dA = [torch.zeros_like(a) for a in A]
    for sm in (-1.0, 1.0):
        for sv in (-1.0, 1.0):
            v = (var.detach() + sv * dvar).clamp_min(rp.MIN_VARIANCE * om.y_std**2)
            try:
                Ap = partials(mu.detach() + sm * dmu, v, c0)
            except RuntimeError:  # a lowered variance can make the joint covariance indefinite: that corner is void
                continue
            dA = [torch.maximum(x, (a - b).abs()) for x, a, b in zip(dA, Ap, A)]
    # sums of absolute terms of the fp32 sums over the training points
    sy, s2 = om.y_std, om.y_std**2
    Xn = rp._normalise(torch.tensor(pts, dtype=torch.float64), om.lo, om.rng)
    T = [torch.zeros(len(pts), d, dtype=torch.float64) for _ in outs]
    Pn = None if pend is None else rp._normalise(torch.tensor(pend, dtype=torch.float64), om.lo, om.rng)
    beta = None
    if Pn is not None:
        kP = rp.kernel_matrix(om.spec, om.Xn, Pn)  # (n, p)
        beta = torch.cholesky_solve(kP, om.L)
    for r in range(len(pts)):
        xr = torch.tensor(pts[r], dtype=torch.float64)
        J = torch.autograd.functional.jacobian(
            lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), om.Xn)[0], xr).abs()  # (n, d)
        k = rp.kernel_matrix(om.spec, Xn[r : r + 1], om.Xn)[0]
        u = torch.cholesky_solve(k[:, None], om.L)[:, 0]
        T[0][r] = sy * om.alpha.abs() @ J
        T[1][r] = 2 * s2 * u.abs() @ J
        if Pn is not None:
            JP = torch.autograd.functional.jacobian(
                lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), Pn)[0], xr).abs()
            for q in range(Pn.shape[0]):
                T[2 + q][r] = s2 * (JP[q] + beta[:, q].abs() @ J)
    eps32 = 2.0**-19 * math.sqrt(om.Xn.shape[0])
    bound = 1e-3 * g_ref.abs() + 1e-7 * sy
    for a, da, g, t in zip(A, dA, grads, T):
        bound = bound + eps32 * a.abs()[:, None] * t + da[:, None] * g
    return bound


SHAPES = [(1, 5, None), (4, 64, 1.7), (20, 256, None)]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"d{d}-n{n}-{'os' if o else 'noos'}" for d, n, o in SHAPES])
def test_gradient_and_value_against_the_oracle_without_pending(family, shape):
    d, n, os_ = shape
    gp, om, X, pts = _setup(family, d, n, os_)
    z = sobol_normal_samples(S, 1, 7)
    worst = 0.0
    for kind in GRAD_KINDS:
        spec, cfg = _acq(kind, om, X)
        zz = z if cfg.is_mc else None
        val, grad = gp.value_and_grad(cfg, torch.from_numpy(pts), zz)
        val2, grad2 = gp.value_and_grad(cfg, torch.from_numpy(pts), zz)
        assert torch.equal(val, val2) and torch.equal(grad, grad2), "repeated calls must be bit-identical"
        # the value agrees with the one the engine reports (gp.score) within score_bounds
        _, bound_v = score_bounds(om, spec, pts, None if zz is None else zz[:, 0])
        scores, _ = gp.score(cfg, torch.from_numpy(pts), None if zz is None else zz[:, 0])
        assert bool(((val.double().cpu() - scores.double().cpu()).abs() <= bound_v).all()), (kind, val, scores)
        _, g_ref = oracle_value_and_grad(om, spec, pts, None if zz is None else zz[:, 0])
        bound = _bound(om, spec, pts, None if zz is None else zz[:, 0], None, g_ref)
        err = (grad.double().cpu() - g_ref).abs()
        worst = max(worst, float((err / bound).max()))
        assert bool((err <= bound).all()), (kind, float((err / bound).max()), err.max())
        if d > 1:
            assert bool((grad[:, 1] == 0).all()), "inactive column"
    print(f"{family} {shape}: worst err/bound {worst:.3f}")


@pytest.mark.parametrize("family", ("matern52", "rbf"))
@pytest.mark.parametrize("p", (1, 8, 31))
def test_gradient_and_value_against_the_oracle_with_pending(family, p):
    gp, om, X, pts = _setup(family, 4, 64, 1.3, seed=p)
    rng = np.random.default_rng(100 + p)
    pend = np.vstack([rng.uniform(0, 1, (p - 1, 4)), pts[:1] + 0.02]).clip(0, 1) if p > 1 else pts[:1] + 0.02
    z = sobol_normal_samples(S, 1 + p, 11)
    worst = 0.0
    for kind in MC:
        spec, cfg = _acq(kind, om, X)
        val, grad = gp.value_and_grad(cfg, torch.from_numpy(pts), z, pend)
        val2, grad2 = gp.value_and_grad(cfg, torch.from_numpy(pts), z, pend)
        assert torch.equal(val, val2) and torch.equal(grad, grad2)
        joint = gp.score_joint(cfg, torch.from_numpy(pts), pend, z).double().cpu()
        g_ref_v, g_ref = oracle_value_and_grad(om, spec, pts, z, pend)
        tol_v = 2e-4 + 2e-3 * g_ref_v.abs()
        assert bool(((val.double().cpu() - joint).abs() <= tol_v).all()), (kind, val, joint)
        assert bool(((val.double().cpu() - g_ref_v).abs() <= tol_v).all()), (kind, val, g_ref_v)
        bound = _bound(om, spec, pts, z, pend, g_ref)
        err = (grad.double().cpu() - g_ref).abs()
        worst = max(worst, float((err / bound).max()))
        assert bool((err <= bound).all()), (kind, float((err / bound).max()), err.max())
    print(f"{family} p={p}: worst err/bound {worst:.3f}")


# ---- optimiser quality ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ("qLogEI", "EI", "UCB"))
def test_continuous_2d_reaches_the_dense_grid_optimum(kind):
    from baybe_b200.continuous import recommend_continuous_hybrid

    gp, om, X, _ = _setup("matern52", 2, 16, None, seed=3)
    spec, cfg = _acq(kind, om, X)
    z = sobol_normal_samples(512, 1, 5)
    cb = np.array([[0.0, 0.0], [1.0, 1.0]])
    pts, idx, value = recommend_continuous_hybrid(gp, cfg, np.zeros((1, 0)), cb, 1, seed=5)
    zz = z[:, 0] if cfg.is_mc else None
    g = np.linspace(0, 1, 201)
    grid = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    gv = oracle.acq_values(om, spec, grid, zz)
    v, gr = oracle_value_and_grad(om, spec, pts, zz)
    scale = max(1.0, float(gv.abs().max()))
    assert float(v[0]) >= float(gv.max()) - 1e-3 * scale, (float(v[0]), float(gv.max()))
    on_bound = (np.abs(pts[0] - cb[0]) < 1e-6) | (np.abs(pts[0] - cb[1]) < 1e-6)
    gproj = np.where(on_bound, 0.0, gr[0].numpy())
    gmax = float(oracle_value_and_grad(om, spec, grid[::97], zz)[1].abs().max())
    assert np.all(np.abs(gproj) <= 2e-2 * max(gmax, 1e-12)), (gproj, gmax)


def test_hybrid_qei_batch_reaches_an_exhaustive_greedy_search():
    from baybe_b200.continuous import recommend_continuous_hybrid

    rng = np.random.default_rng(9)
    disc = np.array([[a, b] for a in (0.0, 0.2, 0.4, 0.6, 0.8, 1.0) for b in (0.0, 1.0)])  # 12 configurations
    n = 24
    X = np.hstack([disc[rng.integers(0, 12, n)], rng.uniform(0, 1, (n, 2))])
    y = np.sin(3 * X[:, 0]) + X[:, 1] - (X[:, 2] - 0.6) ** 2 + np.cos(4 * X[:, 3]) + 0.02 * rng.normal(size=n)
    ls = np.array([0.4, 0.8, 0.35, 0.35])
    bounds = np.array([np.zeros(4), np.ones(4)])
    gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=bounds, family="matern52", lengthscale=ls, noise=1e-3)
    spec_k = oracle.KernelSpec(family="matern52", lengthscale=ls, active_dims=[0, 1, 2, 3])
    om = oracle.build_model(spec_k, X, y, bounds, noise=1e-3)
    spec, cfg = _acq("qEI", om, X)
    cb = np.array([[0.0, 0.0], [1.0, 1.0]])
    pts, idx, value = recommend_continuous_hybrid(gp, cfg, disc, cb, 3, seed=3)
    assert all(np.array_equal(pts[j, :2], disc[idx[j]]) for j in range(3))
    g = np.linspace(0, 1, 41)
    cgrid = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    rows = np.hstack([np.repeat(disc, len(cgrid), 0), np.tile(cgrid, (12, 1))])
    chosen = []
    for j in range(3):
        z = sobol_normal_samples(512, 1 + j, 3)
        v = oracle.acq_values_joint(om, spec, rows, np.array(chosen).reshape(-1, 4), z) if j else \
            oracle.acq_values(om, spec, rows, z[:, 0])
        chosen.append(rows[int(v.argmax())])
    zj = sobol_normal_samples(512, 3, 3)
    ref = float(oracle.acq_values_joint(om, spec, np.array(chosen[:1]), np.array(chosen[1:]), zj)[0])
    ours = float(oracle.acq_values_joint(om, spec, pts[:1], pts[1:], zj)[0])
    assert ours >= ref - 0.01 * abs(ref) - 1e-6, (ours, ref)
    assert value == pytest.approx(ours, rel=2e-3, abs=1e-5)


def test_config3_shape_with_qlogei_q16_runs_and_every_point_is_valid():
    from baybe_b200.continuous import recommend_continuous_hybrid

    rng = np.random.default_rng(2)
    lv = np.linspace(0, 1, 6)
    disc = np.array(np.meshgrid(lv, lv, lv, lv, indexing="ij")).reshape(4, -1).T  # 1296 configurations
    n = 256
    X = np.hstack([disc[rng.integers(0, len(disc), n)], rng.uniform(0, 1, (n, 4))])
    y = np.sin(3 * X).sum(1) + 0.05 * rng.normal(size=n)
    bounds = np.array([np.zeros(8), np.ones(8)])
    gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=bounds, family="matern52", lengthscale=np.full(8, 0.6),
                  noise=1e-3)
    cfg = AcqConfig("qLogEI", best_f=gp.best_f(AcqConfig("qLogEI")))
    cb = np.array([np.zeros(4), np.ones(4)])
    pts, idx, value = recommend_continuous_hybrid(gp, cfg, disc, cb, 16, seed=1)
    assert pts.shape == (16, 8) and np.isfinite(value)
    assert all(np.array_equal(pts[j, :4], disc[idx[j]]) for j in range(16))
    assert np.all(pts[:, 4:] >= 0) and np.all(pts[:, 4:] <= 1)


# ---- Campaign flows on the CUDA engine -----------------------------------------------------------------------------
def test_campaign_flows_on_the_engine():
    pytest.importorskip("tests.test_continuous")
    from tests import test_continuous as tc

    if tc.REF is None:
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    import sys

    for p in (str(tc.ROOT / "tests" / "shims"), str(tc.REF)):
        if p not in sys.path:
            sys.path.append(p)
    from baybe.acquisition import qLogEI

    from baybe_b200 import baybe_plugin

    rng = np.random.default_rng(4)
    for kind, acqf in (("continuous", None), ("hybrid", qLogEI())):
        space = tc._space(kind, fixed=True)
        camp = tc._campaign(baybe_plugin, space, acqf=acqf)
        camp.add_measurements(tc._measure(tc._initial(space, 8, rng), rng))
        rec = camp.recommend(3, pending_experiments=tc._initial(space, 1, rng))
        assert len(rec) == 3 and (rec["flow"] == 2.0).all()
        assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
        vals = camp.acquisition_values(rec)
        assert np.all(np.isfinite(vals.to_numpy(dtype=float)))
        camp.add_measurements(tc._measure(rec, rng))
        assert len(camp.recommend(2)) == 2
