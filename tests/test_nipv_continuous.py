"""CPU tests of qNIPV on continuous and hybrid search spaces: the argument checks of ``bb_nipv_phi`` and
``bb_nipv_grad`` before any CUDA call, the float64 stand-in (tests/nipv_grad_oracle.py) against finite differences and
the definition, ``recommend_continuous_hybrid`` with a ``NipvScorer`` on it, and Campaign flows on the stand-in engine
(tests/nipv_oracle.py behind ``nipv._nipv_score`` and ``nipv._joint_posterior``, tests/nipv_grad_oracle.py behind
``nipv._nipv_phi`` and ``nipv._nipv_grad``)."""
from __future__ import annotations

import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from baybe_b200 import _lib
from baybe_b200 import nipv as nv
from baybe_b200.engine import AcqConfig
from tests import nipv_grad_oracle as go
from tests import nipv_oracle as po
from tests.test_continuous import REF, ROOT, _initial, _measure, _space

needs_ref = pytest.mark.skipif(REF is None, reason="the reference package (baybe) is not installed under oracle/_ref")


# ---- bb_nipv_phi / bb_nipv_grad: argument checks before any CUDA call --------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _fake(case: str):
    from tests.test_abi import _fake_model

    m = _fake_model(case == "wide", 1)
    m.n = m.n_pad = 300 if case == "n 300" else 64
    if case == "task":
        m.task_col = 0
    return m


_PHI_BAD = [
    ("null model", "invalid", b"model struct"),
    ("wide", "unsupported", b"wide-feature"),
    ("task", "unsupported", b"task parameter"),
    ("n 300", "unsupported", b"at most 256"),
    ("M 0", "invalid", b"M=0"),
    ("n_cond -1", "invalid", b"n_cond=-1"),
    ("n_cond 32", "invalid", b"n_cond=32"),
    ("null xm", "invalid", b"null buffer"),
    ("null image", "invalid", b"null buffer"),
    ("null cross", "invalid", b"need cross_m and linv"),
    ("null linv", "invalid", b"need cross_m and linv"),
]


@pytest.mark.parametrize("case, status, msg", _PHI_BAD, ids=[c for c, *_ in _PHI_BAD])
def test_nipv_phi_rejects_bad_arguments_before_any_cuda_call(lib, case, status, msg):
    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    m = _fake(case)
    p = C.c_void_p(1 << 20)
    M = 0 if case == "M 0" else 100
    n_cond = {"n_cond -1": -1, "n_cond 32": 32}.get(case, 2)
    rc = lib.bb_nipv_phi(None if case == "null model" else C.byref(m), None if case == "null xm" else p, M, n_cond,
                         None if case == "null cross" else p, None if case == "null linv" else p,
                         None if case == "null image" else p, None)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


_GRAD_BAD = [
    ("null model", "invalid", b"model struct"),
    ("wide", "unsupported", b"wide-feature"),
    ("task", "unsupported", b"task parameter"),
    ("n 300", "unsupported", b"at most 256"),
    ("P 0", "invalid", b"P=0"),
    ("P -1", "invalid", b"P=-1"),
    ("M 0", "invalid", b"M=0"),
    ("n_cond -1", "invalid", b"n_cond=-1"),
    ("n_cond 32", "invalid", b"n_cond=32"),
    ("null noise", "invalid", b"null noise"),
    ("bad noise", "invalid", b"noise not finite"),
    ("bad prior", "invalid", b"prior_var"),
    ("null x", "invalid", b"null buffer"),
    ("null image", "invalid", b"null buffer"),
    ("null value", "invalid", b"null buffer"),
    ("null grad", "invalid", b"null buffer"),
    ("null workspace", "invalid", b"null buffer"),
    ("null cond_x", "invalid", b"need cond_x"),
    ("null beta", "invalid", b"need cond_x"),
    ("null linv", "invalid", b"need cond_x"),
    ("small workspace", "invalid", b"workspace of"),
]


@pytest.mark.parametrize("case, status, msg", _GRAD_BAD, ids=[c for c, *_ in _GRAD_BAD])
def test_nipv_grad_rejects_bad_arguments_before_any_cuda_call(lib, case, status, msg):
    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    m = _fake(case)
    p = C.c_void_p(1 << 20)
    P = {"P 0": 0, "P -1": -1}.get(case, 10)
    M = 0 if case == "M 0" else 1000
    n_cond = {"n_cond -1": -1, "n_cond 32": 32}.get(case, 2)
    noise = None if case == "null noise" else (C.c_float * 1)(-1.0 if case == "bad noise" else 0.01)
    prior = float("nan") if case == "bad prior" else 1.0
    need = _lib.nipv_grad_ws_bytes(10, 1000, 64, 2, m.d)
    ws_bytes = need - 4 if case == "small workspace" else need
    nul = lambda name: None if case == f"null {name}" else p  # noqa: E731
    rc = lib.bb_nipv_grad(None if case == "null model" else C.byref(m), noise, prior, nul("x"), P, nul("image"), M,
                          n_cond, nul("cond_x"), nul("beta"), nul("linv"), nul("value"), nul("grad"), nul("workspace"),
                          ws_bytes, None)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


def test_nipv_grad_accepts_the_stated_minimum_workspace():
    """The stated minimum: one R = n + n_cond + d + 1 row per point for the point pass and per pair-pass CTA, with at
    most 264 CTAs and one per 64 integration points."""
    assert _lib.nipv_grad_ws_bytes(3, 1, 10, 0, 2) == 4 * 3 * 13 * 2
    assert _lib.nipv_grad_ws_bytes(3, 65, 10, 1, 2) == 4 * 3 * 14 * 3
    assert _lib.nipv_grad_ws_bytes(1, 10**6, 256, 8, 20) == 4 * 285 * 265


# ---- the stand-in against finite differences and the definition --------------------------------------------------------
@pytest.fixture()
def f64_engine(monkeypatch):
    monkeypatch.setattr(nv, "_joint_posterior", po.joint_posterior_f64)
    monkeypatch.setattr(nv, "_nipv_score", po.nipv_score_f64)
    monkeypatch.setattr(nv, "_nipv_phi", go.nipv_phi_f64)
    monkeypatch.setattr(nv, "_nipv_grad", go.nipv_grad_f64)


def _gp(d=2, n=10, seed=0, family="matern52", outputscale=1.3):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (n, d))
    y = np.sin(3 * X).sum(1) + 0.1 * rng.normal(size=n)
    bounds = np.stack([np.zeros(d), np.ones(d)])
    return po.NipvStandInGP(X, y, bounds, family, np.full(d, 0.35), 2e-2, outputscale=outputscale)


def _scorer(gp, M=30, seed=1):
    xm = np.random.default_rng(seed).uniform(0, 1, (M, gp.d)).astype(np.float32).astype(np.float64)
    return nv.NipvScorer(gp, AcqConfig("qNIPV"), xm), xm


@pytest.mark.parametrize("n_cond", [0, 1, 3])
def test_stand_in_matches_finite_differences_and_the_definition(f64_engine, n_cond):
    gp = _gp()
    sc, xm = _scorer(gp)
    rng = np.random.default_rng(4)
    pend = rng.uniform(0, 1, (n_cond, 2)) if n_cond else None
    x = np.array([[0.42, 0.57], [0.8, 0.2], [0.05, 0.95]]).astype(np.float32).astype(np.float64)  # rows go as fp32
    val, g = sc.value_and_grad(torch.from_numpy(x), pend)
    ref = po.nipv_definition(gp, x, xm, pend if n_cond else np.zeros((0, 2)))
    np.testing.assert_allclose(val.numpy(), ref, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(sc.scores(x, pend, 0, 64), ref, rtol=1e-9, atol=1e-12)
    h = 1e-5
    for j in range(2):
        e = np.zeros_like(x)
        e[:, j] = h
        fd = (po.nipv_definition(gp, x + e, xm, pend if n_cond else np.zeros((0, 2)))
              - po.nipv_definition(gp, x - e, xm, pend if n_cond else np.zeros((0, 2)))) / (2 * h)
        np.testing.assert_allclose(g.numpy()[:, j], fd, rtol=1e-5, atol=1e-9)


# ---- recommend_continuous_hybrid with a NipvScorer ---------------------------------------------------------------------
class _Counter:
    def __init__(self, fn):
        self.fn, self.calls = fn, 0

    def __call__(self, *args, **kw):
        self.calls += 1
        return self.fn(*args, **kw)


def test_continuous_q1_reaches_the_dense_grid_optimum(f64_engine):
    from baybe_b200.continuous import recommend_continuous_hybrid

    gp = _gp(n=8, seed=2)
    sc, _ = _scorer(gp, M=40, seed=3)
    pts, idx, value = recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), np.array([[0.0, 0.0], [1.0, 1.0]]),
                                                  1, n_raw_samples=32, n_restarts=4, seed=1)
    g = np.linspace(0, 1, 61)
    grid = np.array(list(itertools.product(g, g)))
    best = sc.scores(grid, None, 0, 64).max()
    assert idx == [0] and (pts >= 0).all() and (pts <= 1).all()
    assert value >= best - 2e-5 * abs(best)
    assert value == pytest.approx(float(sc.scores(pts, None, 0, 64)[0]), rel=1e-12)


def test_hybrid_q3_matches_an_exhaustive_greedy_search(f64_engine, monkeypatch):
    """Discrete column 0 (4 levels) x continuous column 1, fixed column 2: the greedy batch reaches the value of an
    exhaustive greedy search over a dense grid, discrete and fixed columns never move, and each greedy step builds its
    conditioning and image once."""
    from baybe_b200.continuous import recommend_continuous_hybrid

    gp = _gp(d=3, n=12, seed=5)
    sc, _ = _scorer(gp, M=30, seed=6)
    disc = np.array([[0.0], [0.3], [0.6], [1.0]])
    cb = np.array([[0.0, 0.0], [1.0, 1.0]])
    phi, jp = _Counter(nv._nipv_phi), _Counter(nv._joint_posterior)
    monkeypatch.setattr(nv, "_nipv_phi", phi)
    monkeypatch.setattr(nv, "_joint_posterior", jp)
    pts, idx, value = recommend_continuous_hybrid(sc, sc.cfg, disc, cb, 3, n_raw_samples=16, n_restarts=4, seed=2,
                                                  fixed={1: 0.4})
    assert phi.calls == 3  # one image per greedy step
    assert jp.calls == 2 + 1  # steps 2 and 3 condition on the earlier points, then the joint value of the batch
    assert np.allclose(pts[:, 0], disc[idx, 0]) and np.allclose(pts[:, 2], 0.4)
    assert (pts[:, 1] >= 0).all() and (pts[:, 1] <= 1).all()
    g = np.linspace(0, 1, 201)
    cand = np.array([[dv, c, 0.4] for dv in disc[:, 0] for c in g])
    chosen = []
    for _ in range(3):
        v = sc.scores(cand, np.array(chosen) if chosen else None, 0, 64)
        chosen.append(cand[int(np.argmax(v))])
    exhaustive = sc.joint_value(np.array(chosen), None, 0, 64)
    # L-BFGS-B stops at a projected gradient of 1e-5 (scipy's pgtol) on fp32 rows: a few 1e-6 of the value
    assert value >= exhaustive - 2e-5 * abs(exhaustive)
    # the candidate goes as an fp32 row, its pending points as float64 ones
    assert value == pytest.approx(po.batch_definition(gp, pts, sc.xm.numpy().astype(np.float64)), rel=1e-7)


# ---- Campaign flows on the stand-in engine ------------------------------------------------------------------------------
@pytest.fixture()
def bb(monkeypatch, f64_engine):
    import sys

    if REF is None:
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(REF)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe_b200 import baybe_plugin, surrogates

    monkeypatch.setattr(surrogates, "DeviceGP", po.NipvStandInGP)
    return baybe_plugin


def _campaign(plugin, space, acqf, **kw):
    from baybe import Campaign
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    d = len(space.comp_rep_columns)
    hyper = {"lengthscale": np.full(d, 0.5), "noise": 1e-2, "mean_const": 0.0}
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hyper),
                                        acquisition_function=acqf, n_raw_samples=16, n_restarts=3, **kw)
    return Campaign(space, SingleTargetObjective(NumericalTarget("yield")), rec)


def _check_rows(rec, space):
    assert (rec["flow"] == 2.0).all()
    assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
    if "time" in rec:
        assert set(rec.index) <= set(space.discrete.exp_rep.index)
        disc = space.discrete.exp_rep.loc[rec.index]
        assert (rec["time"].to_numpy() == disc["time"].to_numpy()).all()
        assert (rec["solvent"].to_numpy() == disc["solvent"].to_numpy()).all()


@needs_ref
@pytest.mark.parametrize("kind, acq_kw", [
    ("continuous", {"sampling_n_points": 20}),
    ("continuous", {"sampling_n_points": 1}),
    ("hybrid", {}),
    ("hybrid", {"sampling_fraction": 0.5, "sampling_method": "FPS"}),
    ("hybrid", {"sampling_n_points": 1}),
])
def test_campaign_flow(bb, kind, acq_kw):
    from baybe.acquisition import qNegIntegratedPosteriorVariance

    torch.manual_seed(0)
    np.random.seed(0)
    rng = np.random.default_rng(0)
    space = _space(kind, fixed=True)
    camp = _campaign(bb, space, qNegIntegratedPosteriorVariance(**acq_kw))
    camp.add_measurements(_measure(_initial(space, 6, rng), rng))
    rec = camp.recommend(3)
    assert len(rec) == 3 and list(rec.columns) == list(space.discrete.exp_rep.columns) + list(
        space.continuous.parameter_names)
    _check_rows(rec, space)
    assert isinstance(camp.recommender._scorer, nv.NipvScorer)
    camp.add_measurements(_measure(rec, rng))
    pend = rec.iloc[:1]
    rec2 = camp.recommend(3, pending_experiments=pend)
    assert len(rec2) == 3
    _check_rows(rec2, space)
    vals = camp.acquisition_values(rec2, pending_experiments=pend)
    assert len(vals) == 3 and np.all(np.isfinite(vals.to_numpy(dtype=float))) and (vals < 0).all()
    jv = camp.joint_acquisition_value(rec2)
    assert np.isfinite(jv) and jv < 0


@needs_ref
@pytest.mark.parametrize("kind, acq_kw", [("continuous", {"sampling_n_points": 25}), ("hybrid", {}),
                                          ("hybrid", {"sampling_fraction": 0.5, "sampling_method": "FPS"})])
def test_integration_rows_are_baybes_own_draw(bb, monkeypatch, kind, acq_kw):
    from baybe.acquisition import qNegIntegratedPosteriorVariance

    rng = np.random.default_rng(1)
    space = _space(kind, fixed=True)
    acqf = qNegIntegratedPosteriorVariance(**acq_kw)
    camp = _campaign(bb, space, acqf)
    camp.add_measurements(_measure(_initial(space, 6, rng), rng))
    seen = []
    init = nv.NipvScorer.__init__

    def spy(self, gp, cfg, integration):
        seen.append(np.asarray(integration, dtype=np.float64))
        init(self, gp, cfg, integration)

    monkeypatch.setattr(nv.NipvScorer, "__init__", spy)
    np.random.seed(7)
    torch.manual_seed(7)
    camp.recommend(1)
    np.random.seed(7)
    torch.manual_seed(7)
    ref = acqf.get_integration_points(space).to_numpy(dtype=np.float64)
    assert len(seen) == 1
    np.testing.assert_array_equal(seen[0], ref)


@needs_ref
def test_continuous_space_without_sampling_n_points_raises_baybes_error(bb):
    from baybe.acquisition import qNegIntegratedPosteriorVariance

    rng = np.random.default_rng(2)
    space = _space("continuous")
    camp = _campaign(bb, space, qNegIntegratedPosteriorVariance())
    camp.add_measurements(_measure(_initial(space, 6, rng), rng))
    with pytest.raises(ValueError, match="sampling_n_points"):
        camp.recommend(1)


@needs_ref
def test_linear_constraints_and_task_parameters_raise(bb):
    from baybe import Campaign
    from baybe.acquisition import qNegIntegratedPosteriorVariance
    from baybe.constraints import ContinuousLinearConstraint
    from baybe.exceptions import IncompatibilityError
    from baybe.objectives import SingleTargetObjective
    from baybe.parameters import NumericalContinuousParameter, TaskParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    rng = np.random.default_rng(3)
    cont = [NumericalContinuousParameter("temperature", (40.0, 120.0)),
            NumericalContinuousParameter("pressure", (1.0, 5.0))]
    spaces = [
        SearchSpace.from_product(cont, constraints=[ContinuousLinearConstraint(
            parameters=["temperature", "pressure"], operator="<=", coefficients=[1.0, 1.0], rhs=100.0)]),
        SearchSpace.from_product(cont + [TaskParameter("task", values=["a", "b"], active_values=["a"])]),
    ]
    for space, match in zip(spaces, ["constraints", "task parameters"]):
        d = len(space.comp_rep_columns) - (match == "task parameters")  # no lengthscale for the task column
        rec = bb.B200BotorchRecommender(
            surrogate_model=GaussianProcessSurrogate(hyperparameters={"lengthscale": np.full(d, 0.5), "noise": 1e-2,
                                                                      "mean_const": 0.0}),
            acquisition_function=qNegIntegratedPosteriorVariance(sampling_n_points=10), n_raw_samples=16,
            n_restarts=2)
        camp = Campaign(space, SingleTargetObjective(NumericalTarget("yield")), rec)
        init = _initial(_space("continuous"), 6, rng)
        if match == "task parameters":
            init["task"] = ["a", "b"] * 3
        camp.add_measurements(_measure(init, rng))
        with pytest.raises(IncompatibilityError, match=match):
            camp.recommend(1)

