"""CPU tests of desirability objectives and transformed targets on continuous and hybrid search spaces: the argument
checks of ``bb_objective_grad`` before any CUDA call, and Campaign flows on a float64 stand-in engine
(tests/objective_grad_oracle.py behind the ``objectives._objective_grad`` seam, tests/objective_oracle.py behind
``objectives._objective_score``)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

from baybe_b200 import objectives as ob
from tests import objective_oracle as oo
from tests.objective_grad_oracle import StandInObjectiveGP, objective_grad_f64
from tests.test_continuous import REF, _initial, _space

needs_ref = pytest.mark.skipif(REF is None, reason="the reference package (baybe) is not installed under oracle/_ref")


# ---- bb_objective_grad: argument checks before any CUDA call --------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


_BAD = [
    ("null models", "invalid", b"model array is null"),
    ("M = 0", "unsupported", b"n_targets=0"),
    ("M = 9", "unsupported", b"n_targets=9"),
    ("null model entry", "invalid", b"model 1 missing"),
    ("wide", "unsupported", b"wide-feature"),
    ("task", "unsupported", b"task parameter"),
    ("n_pad 512", "unsupported", b"n_pad=512"),
    ("mixed d", "invalid", b"differs from model 0"),
    ("kind 11", "invalid", b"not a single-objective"),
    ("analytic with pending", "invalid", b"analytic kinds take no pending points"),
    ("analytic non-affine", "unsupported", b"affine targets"),
    ("analytic GEOM_MEAN", "unsupported", b"MEAN scalarisation"),
    ("33 pending", "invalid", b"n_pending=33"),
    ("S 0", "invalid", b"S=0"),
    ("S 1025", "invalid", b"S=1025"),
    ("null samples", "invalid", b"null base samples"),
    ("null pending", "invalid", b"pending points need"),
    ("null beta entry", "invalid", b"pending points need"),
    ("null output", "invalid", b"null buffer"),
]


def _grad_call(lib, case: str, N: int = 10):
    from baybe_b200 import _lib
    from baybe_b200.engine import objective_struct
    from tests.test_continuous import _fake

    M = {"M = 0": 0, "M = 9": 9}.get(case, 2)
    ms = [_fake(wide=case == "wide" and m == 1, task=case == "task" and m == 1,
                n_pad=512 if case == "n_pad 512" and m == 1 else 64) for m in range(max(M, 1))]
    if case == "mixed d":
        ms[1].d += 1
    arr = (C.POINTER(_lib.Model) * len(ms))(*(C.pointer(m) for m in ms))
    if case == "null model entry":
        arr[1] = C.POINTER(_lib.Model)()
    kind = {"kind 11": 11, "analytic with pending": 6, "analytic non-affine": 6, "analytic GEOM_MEAN": 6}.get(
        case, _lib.ACQ_KIND["qLogEI"])
    a = _lib.AcqSpec(kind=kind, obj_scale=1.0, tau_relu=1e-6, tau_max=1e-2, tau_pi=1e-3)
    affine = [(_lib.OBJ_OP["AFFINE"], (2.0, 1.0, 0.0))]
    bell = [(_lib.OBJ_OP["BELL"], (0.0, 1.0, 0.0))]
    progs = [bell if case == "analytic non-affine" or kind == 0 else affine] * min(max(M, 1), 8)
    scal = 2 if case == "analytic GEOM_MEAN" or (kind == 0 and M > 1) else (1 if M > 1 else 0)
    obj = objective_struct(min(max(M, 1), 8), scal, progs, [1.0 / max(M, 1)] * min(max(M, 1), 8))
    obj.n_targets = M
    buf = C.c_void_p(1 << 20)
    P = {"analytic with pending": 1, "33 pending": 33, "null pending": 2, "null beta entry": 2}.get(case, 0)
    betas = (C.c_void_p * max(M, 1))(*([1 << 20] * max(M, 1)))
    if case == "null beta entry":
        betas[1] = None
    pend = None if case == "null pending" else buf
    S = {"S 0": 0, "S 1025": 1025}.get(case, 64)
    z = None if case == "null samples" else buf
    out = None if case == "null output" else buf
    return lib.bb_objective_grad(None if case == "null models" else arr, M, C.byref(a), C.byref(obj), buf, N, P, pend,
                                 betas, pend, pend, pend, z, S, out, out, None)


@pytest.mark.parametrize("case, status, msg", _BAD, ids=[c for c, *_ in _BAD])
def test_objective_grad_rejects_bad_arguments_before_any_cuda_call(lib, case, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    rc = _grad_call(lib, case)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


def test_objective_grad_accepts_an_empty_point_set(lib):
    assert _grad_call(lib, "none", N=0) == 0


# ---- Campaign flows on the stand-in engine ---------------------------------------------------------------------------
class _Counter:
    def __init__(self, fn):
        self.fn, self.calls = fn, 0

    def __call__(self, *args, **kw):
        self.calls += 1
        return self.fn(*args, **kw)


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
        monkeypatch.setattr(surrogates, "DeviceGP", StandInObjectiveGP)
        monkeypatch.setattr(ob, "_objective_score", oo.objective_score_f64)
        monkeypatch.setattr(ob, "_objective_grad", objective_grad_f64)
    return baybe_plugin


def _measure(df: pd.DataFrame, rng) -> pd.DataFrame:
    out = df.copy()
    t, pr = out["temperature"], out["pressure"]
    out["yield"] = 50.0 + 0.1 * (t - 40) + 2.0 * pr + rng.normal(0, 0.2, len(out))
    out["purity"] = 98.0 - 0.0008 * (t - 90) ** 2 + 0.3 * pr + rng.normal(0, 0.05, len(out))
    if "time" in out:
        out["yield"] = out["yield"] + 0.5 * out["time"] + (out["solvent"] == "B") * 1.0
    return out


def _objective(which: str):
    from baybe.objectives import DesirabilityObjective, SingleTargetObjective
    from baybe.targets import NumericalTarget

    if which == "geom":
        return DesirabilityObjective([NumericalTarget("yield").clamp(50.0, 70.0).normalize(),
                                      NumericalTarget.match_bell("purity", match_value=98.0, sigma=0.5)])
    if which == "mean":
        return DesirabilityObjective([NumericalTarget("yield"), NumericalTarget("purity", minimize=True)],
                                     scalarizer="MEAN", require_normalization=False, weights=[1.0, 2.0])
    return SingleTargetObjective(NumericalTarget.match_bell("purity", match_value=98.0, sigma=0.5))


def _campaign(plugin, space, which: str):
    from baybe import Campaign
    from baybe.acquisition import ExpectedImprovement

    from baybe_b200.surrogates import GaussianProcessSurrogate

    d = len(space.comp_rep_columns)
    hyper = {"lengthscale": np.full(d, 0.5), "noise": 1e-3, "mean_const": 0.0}
    extra = {"acquisition_function": ExpectedImprovement()} if which == "mean" else {}
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hyper),
                                        n_mc_samples=64, n_raw_samples=16, n_restarts=3, **extra)
    return Campaign(space, _objective(which), rec)


def _check_rows(rec, space):
    assert (rec["flow"] == 2.0).all()
    assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
    if "time" in rec:
        assert set(rec.index) <= set(space.discrete.exp_rep.index)
        disc = space.discrete.exp_rep.loc[rec.index]
        assert (rec["time"].to_numpy() == disc["time"].to_numpy()).all()
        assert (rec["solvent"].to_numpy() == disc["solvent"].to_numpy()).all()


@needs_ref
@pytest.mark.parametrize("which", ["geom", "mean", "bell"])
@pytest.mark.parametrize("kind", ["continuous", "hybrid"])
def test_campaign_flow(bb, monkeypatch, kind, which):
    torch.manual_seed(0)  # the recommender draws its sampler seeds from torch's generator
    np.random.seed(0)  # and the search space samples its initial points from numpy's
    rng = np.random.default_rng(0)
    space = _space(kind, fixed=True)
    camp = _campaign(bb, space, which)
    init = _measure(_initial(space, 6, rng), rng)
    if which == "geom":  # partial measurements: the two models get different n
        init.loc[init.index[:2], "purity"] = np.nan
    camp.add_measurements(init)
    q = 1 if which == "mean" else 3  # analytic EI recommends one point at a time
    rec = camp.recommend(q)
    assert len(rec) == q and list(rec.columns) == list(space.discrete.exp_rep.columns) + list(
        space.continuous.parameter_names)
    _check_rows(rec, space)
    camp.add_measurements(_measure(rec, rng))
    if which != "mean":
        counter = _Counter(ob.pending_conditioning)
        monkeypatch.setattr(ob, "pending_conditioning", counter)
        pend = rec.iloc[:1]
        rec2 = camp.recommend(3, pending_experiments=pend)
        assert len(rec2) == 3
        _check_rows(rec2, space)
        # one conditioning per greedy step (each has pending points), and one for the joint value of the batch
        assert counter.calls == 3 + 1
        vals = camp.acquisition_values(rec2, pending_experiments=pend)
        assert len(vals) == 3 and np.all(np.isfinite(vals.to_numpy(dtype=float)))
        jv = camp.joint_acquisition_value(rec2)
        assert np.isfinite(jv)
    r1 = camp.recommend(1)
    _check_rows(r1, space)
    torch.manual_seed(11)  # the same base samples for every evaluation below
    v1 = camp.acquisition_values(r1)
    assert np.isfinite(float(v1.iloc[0]))
    torch.manual_seed(11)
    assert camp.joint_acquisition_value(r1) == pytest.approx(float(v1.iloc[0]), rel=1e-6, abs=1e-9)


def test_value_and_grad_matches_finite_differences_on_the_stand_in():
    """The seam's stand-in is the autograd of ``ObjectiveScorer.scores``' definition: central differences agree."""
    from baybe_b200.engine import AcqConfig
    from baybe_b200.objectives import CompiledObjective, ObjectiveScorer

    rng = np.random.default_rng(3)
    gps = []
    for m, n in enumerate((9, 12)):
        X = rng.uniform(0, 1, (n, 2))
        gps.append(StandInObjectiveGP(X, np.sin(3 * X).sum(1) + m, np.array([[0.0, 0.0], [1.0, 1.0]]), "matern52",
                                      np.full(2, 0.4), 1e-3, outputscale=1.2))
    comp = CompiledObjective(["a", "b"], [[("BELL", (1.0, 0.7, 0.0))], [("CLAMP", (-0.5, 1.5, 0.0))]], "GEOM_MEAN",
                             [0.5, 0.5])
    sc = ObjectiveScorer(gps, AcqConfig("qLogEI", best_f=0.3), comp)
    old_s, old_g = ob._objective_score, ob._objective_grad
    ob._objective_score, ob._objective_grad = oo.objective_score_f64, objective_grad_f64
    try:
        pend = np.array([[0.3, 0.6]])
        z = sc.base_samples(64, 1, 5)
        x = np.array([[0.42, 0.57], [0.8, 0.2]])
        val, g = sc.value_and_grad(torch.from_numpy(x), pend, z)
        want = sc.scores(x, pend, 5, 64)
        np.testing.assert_allclose(val.double().numpy(), want, rtol=1e-5, atol=1e-6)
        h = 1e-4
        for j in range(2):
            e = np.zeros_like(x)
            e[:, j] = h
            fd = (sc.scores(x + e, pend, 5, 64) - sc.scores(x - e, pend, 5, 64)) / (2 * h)
            np.testing.assert_allclose(g.double().numpy()[:, j], fd, rtol=2e-2, atol=1e-3)
    finally:
        ob._objective_score, ob._objective_grad = old_s, old_g


@needs_ref
def test_pareto_objectives_on_continuous_spaces_still_raise(bb):
    from baybe import Campaign
    from baybe.acquisition import qLogNParEGO
    from baybe.exceptions import IncompatibleAcquisitionFunctionError
    from baybe.objectives import ParetoObjective
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    rng = np.random.default_rng(2)
    space = _space("continuous")
    d = len(space.comp_rep_columns)
    rec = bb.B200BotorchRecommender(
        surrogate_model=GaussianProcessSurrogate(hyperparameters={"lengthscale": np.full(d, 0.5), "noise": 1e-3,
                                                                  "mean_const": 0.0}),
        acquisition_function=qLogNParEGO(), n_mc_samples=64)
    camp = Campaign(space, ParetoObjective([NumericalTarget("yield"), NumericalTarget("purity")]), rec)
    camp.add_measurements(_measure(_initial(space, 6, rng), rng))
    with pytest.raises(IncompatibleAcquisitionFunctionError):
        camp.recommend(1)
