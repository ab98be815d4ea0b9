"""qNIPV's gradient path on the device: bb_nipv_phi + bb_nipv_grad against float64 autograd of the definition
(tests/nipv_grad_oracle.py), against bb_nipv_score, determinism, the argument checks, the continuous optimiser on the
engine, and Campaign flows.

Tolerances, stated before the first run and derived from fp32 arithmetic:

* Values: |IVR - IVR_ref| <= 2e-4 * max IVR_ref over the case, the bound of test_gpu_nipv.py.  Each e_m = k(m,x) -
  phi(m).phi(x) is an r <= 287-term fp32 dot of entries bounded by sqrt(prior variance) with a cancelling result:
  its error is ~ r eps_32 prior ~ 2e-5 prior, and s carries ~ n eps_32 prior; IVR is a sum of squares of e_m over s,
  so its relative error is a few 1e-5 plus the error of the fp32 L^-1 of the model (the posterior tolerance
  VAR_RTOL = 1e-4 of the device posterior), far inside 2e-4.  That relative reading fails where every k_C(m,x) is
  tiny (x far from all M integration points, max IVR ~ 1e-7 of the prior): the error of e_m is absolute, ~ (r + d)
  eps_32 times the prior variance, not relative to e_m.  So the bound carries a floor of VALUE_ATOL = 1e-6 times the
  prior variance (original units), the fp32 resolution of the covariances IVR is made of (DESIGN.md section 4).
  The device value is also compared with bb_nipv_score's, the discrete path's kernel (fp16 hi/lo image, bb_posterior's
  variance in the denominator).  That kernel was measured up to 6e-4 max IVR from the float64 value (RBF, n = 16,
  d = 2, |C| = 8, M = 4096; DESIGN.md section 4), so the two are compared within the bound plus SCORE_RTOL = 1e-3
  max IVR.
* Gradients: |g - g_ref| <= 5e-3 * max |g_ref| over the case, element by element.  The gradient is h - J_x^T w, where h
  sums a_m dk(m,x)/dx over m and J_x^T w goes back through L^-T and L_C^-T: each term carries the e_m error above
  (a few 1e-5 relative) times a reverse pass whose fp32 triangular solve adds ~ n eps_32 cond(L) ~ 1e-4 of its input.
  The two parts cancel to the gradient; at these shapes neither exceeds ~10 max |g|, so the error stays under ~1e-3
  max |g|; the stated bound leaves a factor of 5 for the posterior tolerance.
"""
from __future__ import annotations

import ctypes
import math
import sys

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import DeviceGP
from baybe_b200 import _lib
from baybe_b200.engine import AcqConfig
from baybe_b200.nipv import NipvScorer
from tests.nipv_grad_oracle import ivr_definition

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
VALUE_RTOL = 2e-4
VALUE_ATOL = 1e-6  # times the prior variance in original units
SCORE_RTOL = 1e-3  # bb_nipv_score against the float64 value, as measured
GRAD_RTOL = 5e-3
f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)  # noqa: E731  rows reach the device as fp32


def _setup(family, n, d, outputscale, seed=0, noise=1e-2):
    rng = np.random.default_rng(seed)
    X = f32(rng.uniform(0, 1, (n, d)))
    y = np.sin(4 * X[:, : min(d, 3)]).sum(1) + 0.05 * rng.normal(size=n)
    ls = np.full(d, 0.35 * math.sqrt(max(d, 1)))
    if d > 1:
        ls[1] = 0.0  # an inactive column
    bounds = np.array([np.zeros(d), np.ones(d)])
    gp = DeviceGP(device=DEV, train_x=X, train_y=y, bounds=bounds, family=family, lengthscale=ls, noise=noise,
                  outputscale=outputscale)
    active = [j for j in range(d) if ls[j] > 0]
    spec = oracle.KernelSpec(family=family, lengthscale=ls[active], active_dims=active, outputscale=outputscale)
    om = oracle.build_model(spec, X, y, bounds, noise=noise)
    return gp, om, rng, X


def _noise_fn(om):
    return lambda rows: np.full(len(rows), max(float(om.noise.numpy()[0]), 1e-4)) * om.y_std**2


def _device(sc, x, C):
    """IVR (original units) and its gradient from bb_nipv_phi + bb_nipv_grad for the conditioning rows C."""
    c = sc.conditioned(C, None)
    img = torch.ops.baybe_b200.nipv_phi(sc.xm, c.cross_m, c.linv, sc.gp.handle)
    cond_x, beta = c.cond if c.linv is not None else (None, None)
    xd = torch.from_numpy(x.astype(np.float32)).to(DEV)
    v, g = torch.ops.baybe_b200.nipv_grad(xd, img, sc.M, cond_x, beta, c.linv, sc.gp.handle)
    return v.double().cpu().numpy(), g.double().cpu().numpy()


CASES = [  # family, outputscale, n, d, |C|, M, P
    ("matern12", None, 100, 20, 8, 4096, 10),
    ("matern12", 1.7, 100, 20, 8, 4096, 10),
    ("matern32", None, 100, 20, 8, 4096, 10),
    ("matern32", 0.6, 100, 20, 8, 4096, 10),
    ("matern52", None, 100, 20, 8, 4096, 10),
    ("matern52", 2.5, 100, 20, 8, 4096, 10),
    ("rbf", None, 100, 20, 8, 4096, 10),
    ("rbf", 1.3, 100, 20, 8, 4096, 10),
    ("matern52", None, 16, 2, 0, 1, 1),
    ("matern52", 1.3, 16, 2, 1, 100, 16),
    ("rbf", None, 256, 20, 31, 4096, 17),
    ("matern32", 1.3, 256, 20, 0, 100, 40),
    ("matern52", None, 100, 62, 8, 100, 17),
    ("matern12", 0.8, 100, 62, 31, 1, 40),
    ("rbf", 1.3, 16, 2, 8, 4096, 16),
    ("matern52", 1.3, 100, 20, 8, 60000, 17),  # 938 chunks of 64 over 264 CTAs: several chunks per CTA
]


@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_value_and_gradient_against_the_float64_oracle(case):
    family, os_, n, d, Cn, M, P = case
    gp, om, rng, X = _setup(family, n, d, os_)
    XM = f32(rng.uniform(0, 1, (M, d)))
    C = f32(rng.uniform(0, 1, (Cn, d))) if Cn else None
    near = min(2, P - 1)  # points near training rows probe the small-variance corner
    x = f32(np.vstack([rng.uniform(0, 1, (P - near, d)), X[:near] + 0.01]).clip(0, 1))
    sc = NipvScorer(gp, AcqConfig("qNIPV"), XM)
    v, g = _device(sc, x, C)
    X = torch.from_numpy(x).requires_grad_(True)
    ref = ivr_definition(om, _noise_fn(om), X, XM, C)
    g_ref = torch.autograd.grad(ref.sum(), X)[0].numpy()
    ref = ref.detach().numpy()
    bound = VALUE_RTOL * ref.max() + VALUE_ATOL * (os_ or 1.0) * om.y_std**2
    assert np.abs(v - ref).max() <= bound, (np.abs(v - ref).max(), ref.max())
    assert np.abs(g - g_ref).max() <= GRAD_RTOL * np.abs(g_ref).max(), (np.abs(g - g_ref).max(), np.abs(g_ref).max())
    if d > 1:
        assert (g[:, 1] == 0).all(), "inactive column"
    # the value bb_nipv_score reports for the same rows and conditioning set
    s, _, _ = sc.values(x, C, None)
    s = s.double().cpu().numpy()
    assert np.abs(v - s).max() <= bound + SCORE_RTOL * ref.max(), (np.abs(v - s).max(), bound)
    # bit-identical repeated calls
    v2, g2 = _device(sc, x, C)
    assert np.array_equal(v, v2) and np.array_equal(g, g2)


def test_scorer_value_and_grad_is_qnipv():
    """value_and_grad reports qNIPV (the value of ``scores``) and its gradient, IVR's over M."""
    gp, om, rng, _ = _setup("matern52", 40, 4, 1.2)
    XM = f32(rng.uniform(0, 1, (500, 4)))
    sc = NipvScorer(gp, AcqConfig("qNIPV"), XM)
    pend = f32(rng.uniform(0, 1, (3, 4)))
    x = f32(rng.uniform(0, 1, (7, 4)))
    val, grad = sc.value_and_grad(torch.from_numpy(x), pend)
    s = sc.scores(x, pend, 0, 64)
    ivr, g = _device(sc, x, pend)
    assert np.abs(val.cpu().numpy() - s).max() <= VALUE_RTOL * ivr.max() / 500
    np.testing.assert_allclose(grad.cpu().numpy(), g / 500, rtol=0, atol=1e-12 + 1e-7 * np.abs(g).max())


def test_workspace_and_point_count_below_the_minimum_are_rejected():
    gp, om, rng, _ = _setup("matern52", 32, 3, None)
    XM = torch.from_numpy(f32(rng.uniform(0, 1, (300, 3))).astype(np.float32)).to(DEV)
    img = torch.ops.baybe_b200.nipv_phi(XM, None, None, gp.handle)
    x = torch.from_numpy(f32(rng.uniform(0, 1, (5, 3))).astype(np.float32)).to(DEV)
    lib = _lib.load()
    noise = (ctypes.c_float * 1)(0.01)
    need = _lib.nipv_grad_ws_bytes(5, 300, gp.n, 0, 3)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out_v = torch.full((5,), -7.0, device=DEV)
    out_g = torch.full((5, 3), -7.0, device=DEV)

    def args(P, nbytes):
        return (ctypes.byref(gp.model), noise, 1.0, x.data_ptr(), P, img.data_ptr(), 300, 0, None, None, None,
                out_v.data_ptr(), out_g.data_ptr(), ws.data_ptr(), nbytes, None)

    assert lib.bb_nipv_grad(*args(5, need - 1)) == _lib.BB_ERR_INVALID
    assert lib.bb_nipv_grad(*args(0, need)) == _lib.BB_ERR_INVALID
    torch.cuda.synchronize()
    assert (out_v == -7.0).all() and (out_g == -7.0).all()  # nothing was launched
    assert lib.bb_nipv_grad(*args(5, need)) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(out_v).all() and torch.isfinite(out_g).all()


def test_continuous_2d_reaches_the_dense_grid_optimum():
    from baybe_b200.continuous import recommend_continuous_hybrid

    gp, om, rng, _ = _setup("matern52", 10, 2, 1.0, seed=3, noise=1e-3)
    sc = NipvScorer(gp, AcqConfig("qNIPV"), f32(rng.uniform(0, 1, (400, 2))))
    pts, idx, value = recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), np.array([[0.0, 0.0], [1.0, 1.0]]), 1,
                                                  seed=2)
    g = np.linspace(0, 1, 101)
    grid = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    best = sc.scores(grid, None, 0, 64).max()
    assert value >= best - 1e-3 * abs(best), (value, best)


def test_hybrid_batch_reaches_an_exhaustive_greedy_search():
    from baybe_b200.continuous import recommend_continuous_hybrid

    rng = np.random.default_rng(7)
    disc = np.array([[a, b] for a in (0.0, 0.5, 1.0) for b in (0.0, 0.3, 0.6, 1.0)])  # 12 configurations
    X = f32(rng.uniform(0, 1, (14, 4)))
    y = np.sin(3 * X).sum(1)
    bounds = np.array([np.zeros(4), np.ones(4)])
    gp = DeviceGP(device=DEV, train_x=X, train_y=y, bounds=bounds, family="matern52", lengthscale=np.full(4, 0.5),
                  noise=1e-3)
    XM = f32(np.hstack([disc[rng.integers(0, 12, 600)], rng.uniform(0, 1, (600, 2))]))
    sc = NipvScorer(gp, AcqConfig("qNIPV"), XM)
    cb = np.array([[0.0, 0.0], [1.0, 1.0]])
    pts, idx, value = recommend_continuous_hybrid(sc, sc.cfg, disc, cb, 3, seed=3)
    assert all(np.array_equal(pts[j, :2], disc[idx[j]]) for j in range(3))
    g = np.linspace(0, 1, 21)
    cgrid = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    rows = np.hstack([np.repeat(disc, len(cgrid), 0), np.tile(cgrid, (12, 1))])
    chosen = []
    for _ in range(3):
        v = sc.scores(rows, np.array(chosen) if chosen else None, 0, 64)
        chosen.append(rows[int(np.argmax(v))])
    exhaustive = sc.joint_value(np.array(chosen), None, 0, 64)
    assert value >= exhaustive - 1e-3 * abs(exhaustive), (value, exhaustive)


def test_a_million_integration_points_fit_the_image_cap():
    gp, om, rng, _ = _setup("matern52", 256, 20, 1.3)
    M = 10**6
    XM = f32(rng.uniform(0, 1, (M, 20)))
    sc = NipvScorer(gp, AcqConfig("qNIPV"), XM)
    pend = f32(rng.uniform(0, 1, (8, 20)))
    x = f32(rng.uniform(0, 1, (10, 20)))
    v, g = _device(sc, x, pend)
    s = sc.values(x, pend, None)[0].double().cpu().numpy()
    assert np.isfinite(v).all() and np.isfinite(g).all()
    assert np.abs(v - s).max() <= VALUE_RTOL * s.max()
    with pytest.raises(NotImplementedError, match="GiB"):
        from baybe_b200.engine import nipv_image_numel

        nipv_image_numel(gp, 4 * 10**6, 31)


def test_campaign_flows_on_the_engine():
    from tests import test_continuous as tc

    if tc.REF is None:
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(tc.ROOT / "tests" / "shims"), str(tc.REF)):
        if p not in sys.path:
            sys.path.append(p)
    from baybe.acquisition import qNegIntegratedPosteriorVariance

    from baybe_b200 import baybe_plugin

    rng = np.random.default_rng(4)
    for kind, acqf in (("continuous", qNegIntegratedPosteriorVariance(sampling_n_points=200)),
                       ("hybrid", qNegIntegratedPosteriorVariance())):
        space = tc._space(kind, fixed=True)
        camp = tc._campaign(baybe_plugin, space, acqf=acqf)
        camp.add_measurements(tc._measure(tc._initial(space, 8, rng), rng))
        rec = camp.recommend(3, pending_experiments=tc._initial(space, 1, rng))
        assert len(rec) == 3 and (rec["flow"] == 2.0).all()
        assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
        assert isinstance(camp.recommender._scorer, NipvScorer)
        vals = camp.acquisition_values(rec)
        assert np.all(np.isfinite(vals.to_numpy(dtype=float))) and (vals < 0).all()
        assert np.isfinite(camp.joint_acquisition_value(rec))
        camp.add_measurements(tc._measure(rec, rng))
        assert len(camp.recommend(2)) == 2
