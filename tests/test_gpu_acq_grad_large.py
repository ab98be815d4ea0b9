"""GPU tests of ``bb_acq_grad_large``, the gradient path for single-task models with n_pad > 256 or wide features:
value and gradient against float64 autograd of the oracle (tests/continuous_oracle.py), values against ``gp.score`` /
``gp.score_joint``, agreement with ``bb_acq_grad`` where both apply, determinism, the continuous and hybrid optimiser
against dense oracle searches, and Campaign flows on the engine.

Gradient bound, per row i and column j, with no outlier allowance (test_gpu_continuous.py's):

    |g_ij - g_ref,ij| <= 1e-3 |g_ref,ij| + EPS32(n) * (|A_mu| T_mu + |A_var| T_var + sum_p |A_c,p| T_c,p)_j
                         + sum over the partials A of max_corner |A(mu +- dmu, var +- dvar) - A| * |d moment / dx_j|
                         + 1e-7 * s_y,

with A_mu, A_var, A_c the float64 partials of the value with respect to the moments, dmu / dvar the stated posterior
tolerances of tests/helpers.py, and T the sums of absolute terms the device adds in fp32 over the n training points:
T_mu = s_y sum_i |alpha_i| |dk_i/dx|, T_var = 2 s_y^2 sum_i |u_i| |dk_i/dx| (u = K~^-1 k), T_c,p = s_y^2 (|dk(x, x_p)/dx|
+ sum_i |beta_p,i| |dk_i/dx|).

Growth in n.  Every fp32 sum the kernel forms (k . alpha, the rows of L^-1 k, the columns of L^-T v, k . beta_p and
the reverse pass over the kernel row) has at most n terms.  Its rounding error is at most n u times its sum of
absolute terms (u = 2^-24) and, for rounding errors of random sign, about sqrt(n) u times it.  The bound takes
EPS32(n) = 2^-19 sqrt(n) = 32 sqrt(n) u: 32 units of the random-sign estimate, which reaches the worst case n u at
n = 1024, the largest model.  The T sums grow with n themselves, since every training row adds a term.  The
moment corners do not depend on n: dmu and dvar are stated relative to max |mu| and the prior variance.

Values are held to the oracle's within ``score_bounds`` with its posterior tolerances grown by sqrt(n / 256) past
n = 256 (``_score_bounds_n``; without pending points) or within test_gpu_continuous.py's
2e-4 + 2e-3 |v| plus the value's change at the corners of the stated posterior tolerances (with them), and to gp.score's
or gp.score_joint's within twice that, since each is within the bound of the oracle.  The scoring path has no
Matern-1/2 on wide models (n_pad > 512 or wide by d), so there the value is compared with the oracle only."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import DeviceGP, sobol_normal_samples
from baybe_b200._lib import GRAD_KINDS
from baybe_b200.engine import acq_grad_op
from baybe_b200.synthetic import numeric_grid_workload
from oracle import reference_path as rp
from tests.continuous_oracle import acq_of_moments, oracle_moments, oracle_value_and_grad
from tests.helpers import oracle_model, posterior_tolerances
from tests.test_gpu_continuous import _acq

pytestmark = pytest.mark.gpu

FAMILIES = ("matern12", "matern32", "matern52", "rbf")
MC = ("qLogEI", "qEI", "qUCB", "qSR", "qPI")
S = 128


def _setup(family, d, n, outputscale, seed=0, n_uniform=12):
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
    pts = np.vstack([rng.uniform(0, 1, (n_uniform, d)), X[:near] + 1e-2 * rng.normal(size=(near, d))]).clip(0, 1)
    return gp, om, X, pts


def _bound(om, spec, pts, z, pend, g_ref):
    """The per-(row, column) bound of the module docstring (test_gpu_continuous.py's, with the kernel rows' Jacobians
    formed in forward mode: d passes instead of n)."""
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
            lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), om.Xn)[0], xr,
            vectorize=True, strategy="forward-mode").abs()  # (n, d)
        k = rp.kernel_matrix(om.spec, Xn[r : r + 1], om.Xn)[0]
        u = torch.cholesky_solve(k[:, None], om.L)[:, 0]
        T[0][r] = sy * om.alpha.abs() @ J
        T[1][r] = 2 * s2 * u.abs() @ J
        if Pn is not None:
            JP = torch.autograd.functional.jacobian(
                lambda x: rp.kernel_matrix(om.spec, rp._normalise(x[None], om.lo, om.rng), Pn)[0], xr,
                vectorize=True, strategy="forward-mode").abs()
            for q in range(Pn.shape[0]):
                T[2 + q][r] = s2 * (JP[q] + beta[:, q].abs() @ J)
    eps32 = 2.0**-19 * math.sqrt(om.Xn.shape[0])  # EPS32(n) of the module docstring
    bound = 1e-3 * g_ref.abs() + 1e-7 * sy
    for a, da, g, t in zip(A, dA, grads, T):
        bound = bound + eps32 * a.abs()[:, None] * t + da[:, None] * g
    return bound


def _value_bound(om, spec, pts, z, pend, ref):
    """Bound on |value - oracle value| with pending points: test_gpu_continuous.py's 2e-4 + 2e-3 |v| plus 1.5 times the
    largest change of the value at the corners of the stated posterior tolerances (mu +- dmu, var +- dvar), as
    ``score_bounds`` adds it."""
    with torch.no_grad():
        mu, var, pe = oracle_moments(om, torch.as_tensor(np.asarray(pts), dtype=torch.float64), pend)
        dmu, dvar = posterior_tolerances(om, mu)
        dev = torch.zeros_like(ref)
        for sm in (-1.0, 1.0):
            for sv in (-1.0, 1.0):
                v = (var + sv * dvar).clamp_min(rp.MIN_VARIANCE * om.y_std**2)
                try:
                    c = acq_of_moments(spec, mu + sm * dmu, v, pe, z)
                except RuntimeError:  # a lowered variance can make the joint covariance indefinite: that corner is void
                    continue
                dev = torch.maximum(dev, (c - ref).abs())
    return 2e-4 + 2e-3 * ref.abs() + 1.5 * dev


def _score_bounds_n(om, spec, pts, z):
    """``score_bounds`` with the stated posterior tolerances (dmu, dvar) grown by sqrt(n / 256) past n = 256, as the
    random-sign roundoff of the n-term fp32 sums behind mu and var grows; at n <= 256 it is ``score_bounds``."""
    mu, var = oracle.posterior(om, pts)
    ref = rp.acq_from_moments(spec, mu, var, z)
    dmu, dvar = posterior_tolerances(om, mu)
    g = math.sqrt(max(1.0, om.Xn.shape[0] / 256))
    dev = torch.zeros_like(ref)
    for sm in (-1.0, 1.0):
        for sv in (-1.0, 1.0):
            v = (var + sv * g * dvar).clamp_min(rp.MIN_VARIANCE * om.y_std**2)
            dev = torch.maximum(dev, (rp.acq_from_moments(spec, mu + sm * g * dmu, v, z) - ref).abs())
    return ref, 2e-4 + 1e-4 * ref.abs() + 1.5 * dev

def _large(gp):
    return acq_grad_op(gp.model) is torch.ops.baybe_b200.acq_grad_large


def _check_kinds(gp, om, X, pts, kinds, label, inactive=None):
    """Every kind without pending points: repeats bit-identical, value within score_bounds of gp.score, gradient within
    the module's bound of the oracle.  Returns the worst err / bound."""
    z = sobol_normal_samples(S, 1, 7)
    worst = 0.0
    for kind in kinds:
        spec, cfg = _acq(kind, om, X)
        zz = z if cfg.is_mc else None
        z0 = None if zz is None else zz[:, 0]
        val, grad = gp.value_and_grad(cfg, torch.from_numpy(pts), zz)
        val2, grad2 = gp.value_and_grad(cfg, torch.from_numpy(pts), zz)
        assert torch.equal(val, val2) and torch.equal(grad, grad2), "repeated calls must be bit-identical"
        ref_v, bound_v = _score_bounds_n(om, spec, pts, z0)
        assert bool(((val.double().cpu() - ref_v).abs() <= bound_v).all()), (kind, val, ref_v)
        if not (gp.model.wide and om.spec.family == "matern12"):  # the scoring path's wide kernels have no Matern-1/2
            # each within bound_v of the oracle
            scores, _ = gp.score(cfg, torch.from_numpy(pts), z0)
            assert bool(((val.double().cpu() - scores.double().cpu()).abs() <= 2 * bound_v).all()), (kind, val, scores)
        _, g_ref = oracle_value_and_grad(om, spec, pts, z0)
        bound = _bound(om, spec, pts, z0, None, g_ref)
        err = (grad.double().cpu() - g_ref).abs()
        worst = max(worst, float((err / bound).max()))
        assert bool((err <= bound).all()), (label, kind, float((err / bound).max()), err.max())
        if inactive is not None:
            assert bool((grad[:, inactive] == 0).all()), "inactive column"
    print(f"{label}: worst err/bound {worst:.3f}")
    return worst


SHAPES = [(1, 257, None), (4, 320, 1.7), (20, 512, None), (4, 513, 1.3), (4, 1000, None), (20, 1024, 1.7)]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("shape", SHAPES, ids=[f"d{d}-n{n}-{'os' if o else 'noos'}" for d, n, o in SHAPES])
def test_gradient_and_value_against_the_oracle_without_pending(family, shape):
    d, n, os_ = shape
    gp, om, X, pts = _setup(family, d, n, os_)
    assert _large(gp)
    _check_kinds(gp, om, X, pts, GRAD_KINDS, f"{family} d{d} n{n}", inactive=1 if d > 1 else None)


@pytest.mark.parametrize("family", ("matern32", "matern52", "rbf"))
@pytest.mark.parametrize("n", (320, 1000))
def test_points_on_training_rows(family, n):
    """Training rows themselves, where the posterior variance is about the noise level and cancels in fp32.  Matern-1/2
    is left out: its kernel has a kink at distance 0, where the gradient is not defined."""
    gp, om, X, _ = _setup(family, 4, n, 1.3, seed=2)
    pts = np.vstack([X[:8], X[n // 2 : n // 2 + 4]])
    _check_kinds(gp, om, X, pts, GRAD_KINDS, f"{family} on rows n{n}", inactive=1)


@pytest.mark.parametrize("family", ("matern52", "rbf"))
@pytest.mark.parametrize("p", (1, 8, 31))
def test_gradient_and_value_against_the_oracle_with_pending(family, p):
    gp, om, X, pts = _setup(family, 4, 400, 1.3, seed=p)
    assert _large(gp)
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
        tol_v = _value_bound(om, spec, pts, z, pend, g_ref_v)
        assert bool(((val.double().cpu() - g_ref_v).abs() <= tol_v).all()), (kind, val, g_ref_v)
        assert bool(((val.double().cpu() - joint).abs() <= 2 * tol_v).all()), (kind, val, joint)
        bound = _bound(om, spec, pts, z, pend, g_ref)
        err = (grad.double().cpu() - g_ref).abs()
        worst = max(worst, float((err / bound).max()))
        assert bool((err <= bound).all()), (kind, float((err / bound).max()), err.max())
    print(f"{family} n400 p={p}: worst err/bound {worst:.3f}")


def _wide_d100():
    """test_gpu_wide.py's d100_n200_m52 workload: wide by d (n_pad 256 x d_pad 100 x 4 B > 56 KB)."""
    w = numeric_grid_workload(N=3000, d=100, n=200, seed=11, lengthscale=np.linspace(1.5, 4.0, 100))
    gp = DeviceGP(device="cuda", **w.gp_kwargs())
    assert gp.model.wide == 1 and gp.model.n_pad == 256
    return w, gp, oracle_model(w)


def test_wide_by_d_model_against_the_oracle():
    w, gp, om = _wide_d100()
    assert _large(gp)
    rng = np.random.default_rng(5)
    pts = np.vstack([w.candidates[:10], w.train_x[:4] + 0.02 * rng.normal(size=(4, 100))]).clip(0, 1)
    _check_kinds(gp, om, w.train_x, pts, GRAD_KINDS, "d100_n200_m52")


@pytest.mark.parametrize("p", (1, 8, 31))
def test_wide_by_d_model_with_pending(p):
    w, gp, om = _wide_d100()
    pts = w.candidates[:8]
    pend = w.candidates[100 : 100 + p]
    z = sobol_normal_samples(S, 1 + p, 13)
    worst = 0.0
    for kind in ("qLogEI", "qEI", "qUCB"):
        spec, cfg = _acq(kind, om, w.train_x)
        val, grad = gp.value_and_grad(cfg, torch.from_numpy(pts), z, pend)
        joint = gp.score_joint(cfg, torch.from_numpy(pts), pend, z).double().cpu()
        g_ref_v, g_ref = oracle_value_and_grad(om, spec, pts, z, pend)
        tol_v = _value_bound(om, spec, pts, z, pend, g_ref_v)
        assert bool(((val.double().cpu() - g_ref_v).abs() <= tol_v).all()), (kind, val, g_ref_v)
        assert bool(((val.double().cpu() - joint).abs() <= 2 * tol_v).all()), (kind, val, joint)
        bound = _bound(om, spec, pts, z, pend, g_ref)
        err = (grad.double().cpu() - g_ref).abs()
        worst = max(worst, float((err / bound).max()))
        assert bool((err <= bound).all()), (kind, float((err / bound).max()), err.max())
    print(f"d100_n200_m52 p={p}: worst err/bound {worst:.3f}")


# ---- agreement with bb_acq_grad where both apply ---------------------------------------------------------------------
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("shape", [(1, 5, 0), (4, 64, 8), (20, 256, 0), (4, 200, 31)],
                         ids=["d1-n5", "d4-n64-p8", "d20-n256", "d4-n200-p31"])
def test_agrees_with_bb_acq_grad_on_shared_shapes(family, shape):
    """With d < 32 both kernels form the kernel row, v, u, mu, var and the cross covariances in the same order and take
    the value and its partials from the same device function (acq_point_partials), so the values are bit-identical.
    The gradients differ only by the order of the final sum over the kernel row (sequential in bb_acq_grad, in row
    groups here) and are held to the module's bound around each other."""
    from baybe_b200 import _lib

    d, n, p = shape
    gp, om, X, pts = _setup(family, d, n, 1.3 if n % 2 else None, seed=n)
    assert not _large(gp)
    rng = np.random.default_rng(n)
    pend = rng.uniform(0, 1, (p, d)) if p else None
    z = sobol_normal_samples(S, 1 + p, 3)
    xd = gp.prepare(torch.from_numpy(pts)).to(torch.float32).contiguous()
    extra = tuple(gp.pending_stats(pend)) if p else (None, None, None, None)  # rows, beta, means, covariance
    for kind in GRAD_KINDS if not p else MC:
        spec, cfg = _acq(kind, om, X)
        zf = z.to("cuda", torch.float32).contiguous() if cfg.is_mc else None
        args = (xd, *extra, zf, gp.handle, _lib.ACQ_KIND[kind], cfg.params())
        v0, g0 = torch.ops.baybe_b200.acq_grad(*args)
        v1, g1 = torch.ops.baybe_b200.acq_grad_large(*args)
        v0, g0, v1, g1 = (t.double().cpu() for t in (v0, g0, v1, g1))
        assert torch.equal(v1, v0), (kind, v0, v1)
        z0 = None if zf is None else (z if p else z[:, 0])
        _, g_ref = oracle_value_and_grad(om, spec, pts, z0, pend)
        bound = _bound(om, spec, pts, z0, pend, g_ref)
        assert bool(((g1 - g0).abs() <= bound).all()), (kind, float(((g1 - g0).abs() / bound).max()))


@pytest.mark.parametrize("p", (0, 8, 31))
def test_base_samples_in_global_memory_give_the_shared_memory_result(monkeypatch, p):
    """Base samples stay in global memory only when S (1 + p) does not fit in shared memory beside the point's scratch,
    which real shapes reach only with d_pad in the tens of thousands; BB_ACQ_GRAD_LARGE_Z_GLOBAL=1 takes that path
    here.  Same samples in the same order: the results are bit-identical."""
    gp, om, X, pts = _setup("matern52", 4, 400, 1.3, seed=40 + p)
    pend = np.random.default_rng(p).uniform(0, 1, (p, 4)) if p else None
    z = sobol_normal_samples(1024, 1 + p, 5)
    for kind in MC:
        _, cfg = _acq(kind, om, X)
        v0, g0 = gp.value_and_grad(cfg, torch.from_numpy(pts), z, pend)
        monkeypatch.setenv("BB_ACQ_GRAD_LARGE_Z_GLOBAL", "1")
        v1, g1 = gp.value_and_grad(cfg, torch.from_numpy(pts), z, pend)
        monkeypatch.delenv("BB_ACQ_GRAD_LARGE_Z_GLOBAL")
        assert torch.equal(v0, v1) and torch.equal(g0, g1), kind


# ---- optimiser quality ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ("qLogEI", "EI", "UCB"))
def test_continuous_2d_reaches_the_dense_grid_optimum_at_n400(kind):
    from baybe_b200.continuous import recommend_continuous_hybrid

    gp, om, X, _ = _setup("matern52", 2, 400, None, seed=3)
    assert _large(gp)
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


def test_hybrid_qei_batch_on_a_wide_model_reaches_an_exhaustive_greedy_search():
    """12 configurations of a 98-column descriptor encoding and 2 continuous parameters, n = 200: the model is wide by
    d (n_pad 256 x d_pad 100 x 4 B > 56 KB)."""
    from baybe_b200.continuous import recommend_continuous_hybrid

    rng = np.random.default_rng(9)
    disc = rng.uniform(0, 1, (12, 98))
    n = 200
    X = np.hstack([disc[rng.integers(0, 12, n)], rng.uniform(0, 1, (n, 2))])
    y = (np.sin(3 * X[:, 0]) + X[:, 1] - (X[:, 98] - 0.6) ** 2 + np.cos(4 * X[:, 99])
         + 0.02 * rng.normal(size=n))
    ls = np.concatenate([np.full(98, 2.5), [0.35, 0.35]])
    bounds = np.array([np.zeros(100), np.ones(100)])
    gp = DeviceGP(device="cuda", train_x=X, train_y=y, bounds=bounds, family="matern52", lengthscale=ls, noise=1e-3)
    assert gp.model.wide == 1 and _large(gp)
    spec_k = oracle.KernelSpec(family="matern52", lengthscale=ls, active_dims=list(range(100)))
    om = oracle.build_model(spec_k, X, y, bounds, noise=1e-3)
    spec, cfg = _acq("qEI", om, X)
    cb = np.array([[0.0, 0.0], [1.0, 1.0]])
    pts, idx, value = recommend_continuous_hybrid(gp, cfg, disc, cb, 3, seed=3)
    assert all(np.array_equal(pts[j, :98], disc[idx[j]]) for j in range(3))
    g = np.linspace(0, 1, 41)
    cgrid = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    rows = np.hstack([np.repeat(disc, len(cgrid), 0), np.tile(cgrid, (12, 1))])
    chosen = []
    for j in range(3):
        z = sobol_normal_samples(512, 1 + j, 3)
        v = oracle.acq_values_joint(om, spec, rows, np.array(chosen).reshape(-1, 100), z) if j else \
            oracle.acq_values(om, spec, rows, z[:, 0])
        chosen.append(rows[int(v.argmax())])
    zj = sobol_normal_samples(512, 3, 3)
    ref = float(oracle.acq_values_joint(om, spec, np.array(chosen[:1]), np.array(chosen[1:]), zj)[0])
    ours = float(oracle.acq_values_joint(om, spec, pts[:1], pts[1:], zj)[0])
    assert ours >= ref - 0.01 * abs(ref) - 1e-6, (ours, ref)
    assert value == pytest.approx(ours, rel=2e-3, abs=1e-5)


# ---- Campaign flows on the CUDA engine -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tc():
    from tests import test_continuous as tc

    if tc.REF is None:
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    import sys

    for p in (str(tc.ROOT / "tests" / "shims"), str(tc.REF)):
        if p not in sys.path:
            sys.path.append(p)
    return tc


@pytest.mark.parametrize("n", (300, 1024))
def test_continuous_qlogei_campaign_past_256_measurements(tc, n):
    from baybe_b200 import baybe_plugin

    rng = np.random.default_rng(n)
    space = tc._space("continuous", fixed=True)
    camp = tc._campaign(baybe_plugin, space)
    camp.add_measurements(tc._measure(tc._initial(space, n, rng), rng))
    for q in (1, 3):
        rec = camp.recommend(q)
        assert len(rec) == q and (rec["flow"] == 2.0).all()
        assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
        assert np.all(np.isfinite(camp.acquisition_values(rec).to_numpy(dtype=float)))


def test_hybrid_campaign_on_a_model_wide_by_d(tc):
    from baybe.parameters import CategoricalParameter

    from baybe_b200 import baybe_plugin

    rng = np.random.default_rng(7)
    base = tc._space("continuous")
    from baybe.searchspace import SearchSpace

    space = SearchSpace.from_product([CategoricalParameter("substance", values=[f"s{i}" for i in range(100)],
                                                           encoding="OHE")] + list(base.continuous.parameters))
    assert len(space.comp_rep_columns) == 102
    camp = tc._campaign(baybe_plugin, space)
    df = tc._initial(space, 140, rng)
    camp.add_measurements(tc._measure(df, rng))
    rec = camp.recommend(3)
    assert len(rec) == 3 and rec["substance"].isin([f"s{i}" for i in range(100)]).all()
    assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
    assert np.all(np.isfinite(camp.acquisition_values(rec).to_numpy(dtype=float)))
