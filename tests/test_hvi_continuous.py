"""CPU tests of qEHVI / qLogEHVI on continuous and hybrid search spaces: the argument checks of ``bb_hvi_grad`` before
any CUDA call, the float64 stand-in (tests/hvi_grad_oracle.py) against finite differences and tests/test_mo.py's
``_hvi_score_f64``, the qLogEHVI reporter's chain rule, one set of pending decompositions per greedy step, the
optimiser against a dense grid and an exhaustive greedy search, and Campaign flows on the stand-in engine (the
stand-in behind the ``multiobjective._hvi_grad`` seam, ``_hvi_score_f64`` behind ``multiobjective._hvi_score``)."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest
import torch

from baybe_b200 import multiobjective as mo
from tests.hvi_grad_oracle import StandInHviGP, hvi_grad_f64
from tests.test_continuous import REF, _initial, _space
from tests.test_mo import _hvi_score_f64

needs_ref = pytest.mark.skipif(REF is None, reason="the reference package (baybe) is not installed under oracle/_ref")


# ---- bb_hvi_grad: argument checks before any CUDA call -------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


_BAD = [
    ("null spec", "invalid", b"acquisition spec is null"),
    ("kind 0", "invalid", b"not a hypervolume acquisition function"),
    ("tau 0", "invalid", b"tau_relu > 0 and tau_max > 0"),
    ("M = 1", "unsupported", b"n_targets=1"),
    ("M = 5", "unsupported", b"n_targets=5"),
    ("null models", "invalid", b"model array is null"),
    ("null scale", "invalid", b"null objective scale/shift"),
    ("null model entry", "invalid", b"model 1 missing"),
    ("wide", "unsupported", b"wide-feature"),
    ("task", "unsupported", b"task parameter"),
    ("n_pad 512", "unsupported", b"n_pad=512"),
    ("mixed d", "invalid", b"differs from model 0"),
    ("negative N", "invalid", b"negative point count"),
    ("33 pending", "invalid", b"n_pending=33"),
    ("S 0", "invalid", b"S=0"),
    ("S 1025", "invalid", b"S=1025"),
    ("cell_stride 0", "unsupported", b"cell_stride=0"),
    ("cell_stride 1025", "unsupported", b"cell_stride=1025"),
    ("null pending", "invalid", b"pending points need"),
    ("null beta entry", "invalid", b"pending points need"),
    ("null samples", "invalid", b"null buffer"),
    ("null cells", "invalid", b"null buffer"),
    ("null output", "invalid", b"null buffer"),
]


def _grad_call(lib, case: str, N: int = 10):
    from baybe_b200 import _lib
    from tests.test_continuous import _fake

    M = {"M = 1": 1, "M = 5": 5}.get(case, 2)
    ms = [_fake(wide=case == "wide" and m == 1, task=case == "task" and m == 1,
                n_pad=512 if case == "n_pad 512" and m == 1 else 64) for m in range(M)]
    if case == "mixed d":
        ms[1].d += 1
    arr = (C.POINTER(_lib.Model) * M)(*(C.pointer(m) for m in ms))
    if case == "null model entry":
        arr[1] = C.POINTER(_lib.Model)()
    kind = 0 if case == "kind 0" else _lib.ACQ_KIND["qLogEHVI"]
    a = _lib.AcqSpec(kind=kind, obj_scale=1.0, tau_relu=0.0 if case == "tau 0" else 1e-6, tau_max=1e-2)
    fa = (C.c_float * M)(*([1.0] * M))
    buf = C.c_void_p(1 << 20)
    P = {"33 pending": 33, "null pending": 2, "null beta entry": 2}.get(case, 0)
    betas = (C.c_void_p * M)(*([1 << 20] * M))
    if case == "null beta entry":
        betas[1] = None
    pend = None if case == "null pending" else buf
    S = {"S 0": 0, "S 1025": 1025}.get(case, 64)
    stride = {"cell_stride 0": 0, "cell_stride 1025": 1025}.get(case, 8)
    z = None if case == "null samples" else buf
    cells = None if case == "null cells" else buf
    out = None if case == "null output" else buf
    return lib.bb_hvi_grad(None if case == "null models" else arr, M, None if case == "null spec" else C.byref(a),
                           None if case == "null scale" else fa, fa, buf, -1 if case == "negative N" else N, P, pend,
                           betas, pend, pend, z, S, cells, cells, cells, stride, out, out, None)


@pytest.mark.parametrize("case, status, msg", _BAD, ids=[c for c, *_ in _BAD])
def test_hvi_grad_rejects_bad_arguments_before_any_cuda_call(lib, case, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    rc = _grad_call(lib, case)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


def test_hvi_grad_accepts_an_empty_point_set(lib):
    assert _grad_call(lib, "none", N=0) == 0


# ---- the stand-in and the scorer's gradient path ----------------------------------------------------------------------
@pytest.fixture()
def seams(monkeypatch):
    monkeypatch.setattr(mo, "_hvi_score", _hvi_score_f64)
    monkeypatch.setattr(mo, "_hvi_grad", hvi_grad_f64)


def _models(d=2, ns=(9, 12), seed=3):
    rng = np.random.default_rng(seed)
    gps = []
    for m, n in enumerate(ns):
        X = rng.uniform(0, 1, (n, d))
        y = np.sin(3 * X).sum(1) * (1 if m % 2 == 0 else -1) + 0.3 * m + 0.05 * rng.normal(size=n)
        gps.append(StandInHviGP(X, y, np.array([np.zeros(d), np.ones(d)]), "matern52", np.full(d, 0.4), 1e-3,
                                outputscale=1.2))
    return gps


def _scorer(kind: str, gps):
    from baybe_b200.engine import AcqConfig
    from baybe_b200.multiobjective import HviScorer

    M = len(gps)
    a = np.array([1.0, -1.0, 1.0, -1.0][:M])
    b = np.array([0.0, 2.0, 0.0, 2.0][:M])
    X0 = np.random.default_rng(11).uniform(0, 1, (8, gps[0].d))
    front = np.stack([gp.posterior(X0)[0].double().numpy() for gp in gps], 1) * a + b
    ref = mo.compute_ref_point(front)
    return HviScorer(gps, AcqConfig(kind=kind), a, b, ref, front)


@pytest.mark.parametrize("kind", ["qEHVI", "qLogEHVI"])
@pytest.mark.parametrize("P", [0, 2])
def test_stand_in_matches_finite_differences_and_the_score_stand_in(seams, kind, P):
    """value_and_grad on the stand-in gives what ``scores`` (``_hvi_score_f64`` through the reporter) gives, and its
    gradient agrees with central differences of ``scores``."""
    sc = _scorer(kind, _models())
    rng = np.random.default_rng(5)
    pend = rng.uniform(0, 1, (P, 2)) if P else None
    z = sc.base_samples(64, P, 5)
    x = np.array([[0.42, 0.57], [0.8, 0.2], [0.15, 0.9]])
    val, g = sc.value_and_grad(torch.from_numpy(x), pend, z)
    want = sc.scores(x, pend, 5, 64)
    np.testing.assert_allclose(val.numpy(), want, rtol=1e-5, atol=1e-6)
    h = 1e-5
    for j in range(2):
        e = np.zeros_like(x)
        e[:, j] = h
        fd = (sc.scores(x + e, pend, 5, 64) - sc.scores(x - e, pend, 5, 64)) / (2 * h)
        np.testing.assert_allclose(g.numpy()[:, j], fd, rtol=2e-2, atol=1e-4 * max(1.0, float(np.abs(fd).max())))


def test_qlogehvi_reporter_chain_rule_with_a_positive_pending_gain(seams):
    """With pending points that improve on the front, the reported value is logaddexp(log gain, v) and its gradient
    is the kernel's times sigmoid(v - log gain)."""
    sc = _scorer("qLogEHVI", _models())
    pend = np.array([[0.1, 0.1], [0.9, 0.5], [0.5, 0.95]])
    z = sc.base_samples(64, 3, 2)
    zz = torch.as_tensor(z, dtype=torch.float64).reshape(-1, sc.M * 4)
    gain = sc._pending_parts(pend, zz)[4]
    assert gain > 0.0
    x = np.array([[0.3, 0.6], [0.7, 0.25]])
    val, g = sc.value_and_grad(torch.from_numpy(x), pend, z)
    stats, linv, w, decomps, _ = sc._pending_parts(pend, zz)
    lower, upper, counts = sc._device_cells(decomps)
    v_raw, g_raw = hvi_grad_f64(sc.gps, torch.from_numpy(x), stats[0][0], [], linv, w, zz.float(), lower, upper,
                                counts, 12, sc.cfg.params(), sc.a, sc.b)
    v_raw, g_raw = v_raw.double(), g_raw.double()
    np.testing.assert_allclose(val.numpy(), np.logaddexp(math.log(gain), v_raw.numpy()), rtol=1e-6)
    np.testing.assert_allclose(g.numpy(), (g_raw * torch.sigmoid(v_raw - math.log(gain))[:, None]).numpy(),
                               rtol=1e-6, atol=1e-12)
    assert float(torch.sigmoid(v_raw - math.log(gain)).min()) < 0.999  # the factor is not trivially 1


def test_pending_decompositions_are_built_once_per_greedy_step(seams, monkeypatch):
    from baybe_b200.continuous import recommend_continuous_hybrid

    sc = _scorer("qEHVI", _models())
    calls = {"n": 0}
    real = mo.box_decomposition

    def counted(*args, **kw):
        calls["n"] += 1
        return real(*args, **kw)

    monkeypatch.setattr(mo, "box_decomposition", counted)
    S = 32
    stats = {}
    pts, _, _ = recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), np.array([[0.0, 0.0], [1.0, 1.0]]), 3,
                                            n_samples=S, seed=1, n_raw_samples=16, n_restarts=3, stats=stats)
    assert pts.shape == (3, 2)
    assert stats["grad_calls"] > 3  # many L-BFGS-B evaluations per step
    # steps 2 and 3 each have pending points (S decompositions once), then the joint value of the batch
    assert calls["n"] == 3 * S


@pytest.mark.parametrize("kind", ["qEHVI", "qLogEHVI"])
def test_continuous_optimum_reaches_the_dense_grid_optimum(seams, kind):
    from baybe_b200.continuous import recommend_continuous_hybrid

    sc = _scorer(kind, _models())
    g = np.linspace(0, 1, 61)
    grid = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    best = float(sc.scores(grid, None, 4, 64).max())
    pts, _, value = recommend_continuous_hybrid(sc, sc.cfg, np.zeros((1, 0)), np.array([[0.0, 0.0], [1.0, 1.0]]), 1,
                                                n_samples=64, seed=4, n_raw_samples=32, n_restarts=6)
    assert value >= best - 1e-6 * max(1.0, abs(best))


def test_hybrid_greedy_batch_matches_an_exhaustive_greedy_search(seams):
    """Three discrete configurations (the first column) x one continuous column: every greedy step of the engine's
    batch is at least as good as the best of the configurations x a dense grid given the same pending points."""
    from baybe_b200.continuous import recommend_continuous_hybrid

    sc = _scorer("qEHVI", _models())
    disc = np.array([[0.1], [0.5], [0.9]])
    pts, idx, _ = recommend_continuous_hybrid(sc, sc.cfg, disc, np.array([[0.0], [1.0]]), 2, n_samples=64, seed=6,
                                              n_raw_samples=24, n_restarts=6)
    g = np.linspace(0, 1, 201)
    cand = np.concatenate([np.repeat(disc, len(g), 0), np.tile(g, 3)[:, None]], 1)
    for step in range(2):
        pend = pts[:step] if step else None
        best = float(sc.scores(cand, pend, 6, 64).max())
        got = float(sc.scores(pts[step: step + 1], pend, 6, 64)[0])
        assert got >= best - 1e-6 * max(1.0, abs(best)), (step, got, best)
        assert pts[step, 0] == disc[idx[step], 0]


# ---- Campaign flows on the stand-in engine ---------------------------------------------------------------------------
@pytest.fixture()
def bb(monkeypatch):
    import sys

    from tests.test_continuous import ROOT

    for p in (str(ROOT / "tests" / "shims"), str(REF)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe_b200 import baybe_plugin, surrogates

    if not torch.cuda.is_available():
        monkeypatch.setattr(surrogates, "DeviceGP", StandInHviGP)
        monkeypatch.setattr(mo, "_hvi_score", _hvi_score_f64)
        monkeypatch.setattr(mo, "_hvi_grad", hvi_grad_f64)
    return baybe_plugin


def _measure(df, rng):
    out = df.copy()
    t, pr = out["temperature"], out["pressure"]
    out["yield"] = 50.0 + 0.1 * (t - 40) + 2.0 * pr + rng.normal(0, 0.2, len(out))
    out["cost"] = 3.0 + 0.0008 * (t - 60) ** 2 + 0.6 * pr + rng.normal(0, 0.05, len(out))
    if "time" in out:
        out["yield"] = out["yield"] + 0.5 * out["time"] + (out["solvent"] == "B") * 1.0
    return out


def pareto_campaign(plugin, space, acqf, targets=None, **kw):
    """Shared with the GPU tests: yield maximised, cost minimised."""
    from baybe import Campaign
    from baybe.objectives import ParetoObjective
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    d = len(space.comp_rep_columns) - (getattr(space, "task_idx", None) is not None)  # the task column has none
    hyper = {"lengthscale": np.full(d, 0.5), "noise": 1e-3, "mean_const": 0.0}
    targets = targets or [NumericalTarget("yield"), NumericalTarget("cost", minimize=True)]
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hyper),
                                        acquisition_function=acqf, n_mc_samples=64, n_raw_samples=16, n_restarts=3,
                                        **kw)
    return Campaign(space, ParetoObjective(targets), rec)


def _check_rows(rec, space):
    assert list(rec.columns) == list(space.discrete.exp_rep.columns) + list(space.continuous.parameter_names)
    assert (rec["flow"] == 2.0).all()
    assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
    if "time" in rec:
        assert set(rec.index) <= set(space.discrete.exp_rep.index)
        disc = space.discrete.exp_rep.loc[rec.index]
        assert (rec["time"].to_numpy() == disc["time"].to_numpy()).all()
        assert (rec["solvent"].to_numpy() == disc["solvent"].to_numpy()).all()


def campaign_flow(plugin, kind: str, acq: str):
    """q = 1, q = 3, pending experiments, acquisition_values and joint_acquisition_value (shared with the GPU
    tests)."""
    from baybe.acquisition.acqfs import qExpectedHypervolumeImprovement, qLogExpectedHypervolumeImprovement

    torch.manual_seed(0)  # the recommender draws its sampler seeds from torch's generator
    np.random.seed(0)  # and the search space samples its initial points from numpy's
    rng = np.random.default_rng(0)
    space = _space(kind, fixed=True)
    acqf = qExpectedHypervolumeImprovement() if acq == "qEHVI" else qLogExpectedHypervolumeImprovement()
    camp = pareto_campaign(plugin, space, acqf)
    camp.add_measurements(_measure(_initial(space, 6, rng), rng))
    r1 = camp.recommend(1)
    assert len(r1) == 1
    _check_rows(r1, space)
    rec = camp.recommend(3)
    assert len(rec) == 3
    _check_rows(rec, space)
    camp.add_measurements(_measure(rec, rng))
    pend = rec.iloc[:1]
    rec2 = camp.recommend(2, pending_experiments=pend)
    assert len(rec2) == 2
    _check_rows(rec2, space)
    vals = camp.acquisition_values(rec2, pending_experiments=pend)
    assert len(vals) == 2 and np.all(np.isfinite(vals.to_numpy(dtype=float)))
    assert np.isfinite(camp.joint_acquisition_value(rec2))
    torch.manual_seed(11)  # the same base samples for both evaluations below
    v1 = camp.acquisition_values(rec2.iloc[:1])
    torch.manual_seed(11)
    assert camp.joint_acquisition_value(rec2.iloc[:1]) == pytest.approx(float(v1.iloc[0]), rel=1e-6, abs=1e-9)


@needs_ref
@pytest.mark.parametrize("acq", ["qEHVI", "qLogEHVI"])
@pytest.mark.parametrize("kind", ["continuous", "hybrid"])
def test_campaign_flow(bb, kind, acq):
    campaign_flow(bb, kind, acq)


@needs_ref
def test_what_still_raises_on_continuous_and_hybrid_spaces(bb):
    from baybe.acquisition.acqfs import qExpectedHypervolumeImprovement, qLogExpectedHypervolumeImprovement
    from baybe.constraints import ContinuousLinearConstraint
    from baybe.exceptions import IncompatibilityError, IncompatibleAcquisitionFunctionError
    from baybe.parameters import NumericalContinuousParameter, TaskParameter
    from baybe.searchspace import SearchSpace, SubspaceContinuous
    from baybe.targets import NumericalTarget

    rng = np.random.default_rng(1)
    space = _space("continuous")
    init = _measure(_initial(space, 6, rng), rng)
    camp = pareto_campaign(bb, space, qExpectedHypervolumeImprovement(alpha=0.1))
    camp.add_measurements(init)
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="alpha"):
        camp.recommend(1)
    names = ["yield", "cost", "t3", "t4", "t5"]
    many = init.assign(t3=1.0, t4=2.0, t5=3.0)
    camp = pareto_campaign(bb, space, qLogExpectedHypervolumeImprovement(), [NumericalTarget(n) for n in names])
    camp.add_measurements(many)
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="2 to 4 targets"):
        camp.recommend(1)
    camp = pareto_campaign(bb, space, qLogExpectedHypervolumeImprovement(),
                           [NumericalTarget("yield"), NumericalTarget.match_bell("cost", match_value=3.5, sigma=0.5)])
    camp.add_measurements(init)
    with pytest.raises(NotImplementedError, match="not affine"):  # as on discrete spaces
        camp.recommend(1)
    cons = ContinuousLinearConstraint(parameters=["temperature", "pressure"], operator="<=", coefficients=[1.0, 1.0],
                                      rhs=100.0)
    cspace = SearchSpace(continuous=SubspaceContinuous(space.continuous.parameters, constraints_lin_ineq=[cons]))
    camp = pareto_campaign(bb, cspace, qEHVI := qExpectedHypervolumeImprovement())
    camp.add_measurements(init)
    with pytest.raises(IncompatibilityError, match="constraints"):
        camp.recommend(1)
    tspace = SearchSpace.from_product([NumericalContinuousParameter("temperature", (40.0, 120.0)),
                                       NumericalContinuousParameter("pressure", (1.0, 5.0)),
                                       TaskParameter("lab", values=["a", "b"], active_values=["a"])])
    camp = pareto_campaign(bb, tspace, qEHVI)
    camp.add_measurements(init.assign(lab="a"))
    with pytest.raises((IncompatibilityError, IncompatibleAcquisitionFunctionError, NotImplementedError)):
        camp.recommend(1)
