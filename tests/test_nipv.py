"""qNIPV without a GPU: the spec (fields, defaults, validator), the Random integration points against the reference's
draw, the engine config, the rejections made before any model is fitted, the argument checks of bb_nipv_score before
any CUDA call, the scorer's values, joint values and greedy batches against the float64 definition on a stand-in
engine (tests/nipv_oracle.py), and Campaign flows on that engine."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest
import torch

from baybe_b200 import _lib
from baybe_b200.acquisition import IncompatibleAcquisitionFunctionError, convert_acqf, qNegIntegratedPosteriorVariance, qNIPV
from baybe_b200.engine import AcqConfig

ROOT = Path(__file__).resolve().parents[1]


def test_spec_fields_defaults_and_validator():
    a = qNIPV()
    assert (a.sampling_n_points, a.sampling_fraction, a.sampling_method) == (None, 1.0, "Random")
    assert qNIPV(sampling_n_points=5).sampling_fraction is None
    assert qNIPV(sampling_fraction=0.25).sampling_fraction == 0.25
    with pytest.raises(ValueError):
        qNIPV(sampling_n_points=5, sampling_fraction=0.5)
    for bad in (0.0, 1.5):
        with pytest.raises(ValueError):
            qNIPV(sampling_fraction=bad)
    with pytest.raises(ValueError):
        qNIPV(sampling_n_points=0)
    assert qNIPV is qNegIntegratedPosteriorVariance and convert_acqf("qNIPV") == qNIPV()
    assert convert_acqf("qNegIntegratedPosteriorVariance") == qNIPV()
    assert qNIPV().supports_batching and qNIPV().supports_pending_experiments


def test_engine_config():
    cfg = AcqConfig("qNIPV")
    assert cfg.is_mc
    with pytest.raises(NotImplementedError):
        cfg.to_c()


def _space(n_rows: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    comp = pd.DataFrame(rng.random((n_rows, 3)), columns=["a", "b", "c"], index=rng.permutation(n_rows) + 100)
    return SimpleNamespace(discrete=SimpleNamespace(comp_rep=comp, is_empty=False),
                           continuous=SimpleNamespace(is_empty=True), comp_rep_columns=("a", "b", "c"))


@pytest.mark.parametrize("kw", [dict(sampling_n_points=7), dict(sampling_n_points=23), dict(sampling_fraction=0.3),
                                dict(), dict(sampling_n_points=10)])
def test_random_integration_points_match_the_reference(kw):
    ref_dir = ROOT / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    from baybe.acquisition import qNIPV as RefNIPV

    space = _space(10)
    np.random.seed(3)
    ref = RefNIPV(**kw).get_integration_points(space)
    np.random.seed(3)
    got = qNIPV(**kw).get_integration_points(space)
    assert list(got.index) == list(ref.index)
    assert np.array_equal(got.to_numpy(), ref.to_numpy())


def test_repeat_and_ceil_rules():
    space = _space(10)
    got = qNIPV(sampling_n_points=23).get_integration_points(space)
    assert len(got) == 23 and list(got.index[:20]) == list(space.discrete.comp_rep.index) * 2
    assert len(qNIPV(sampling_fraction=0.31).get_integration_points(space)) == 4
    with pytest.raises(NotImplementedError):
        qNIPV(sampling_method="FPS").get_integration_points(space)


def _objective(kind="single", transformation=None):
    target = SimpleNamespace(name="y", transformation=transformation)
    if kind == "pareto":
        return SimpleNamespace(is_multi_output=True, targets=[target, target])
    cls = type("DesirabilityObjective" if kind == "desirability" else "SingleTargetObjective", (), {})
    obj = cls()
    obj.is_multi_output, obj.targets = False, [target]
    return obj


def test_rejections_before_the_fit():
    from baybe_b200.multiobjective import _error

    space = _space(10)
    space.type = SimpleNamespace(name="DISCRETE")
    fitted = []
    surrogate = SimpleNamespace(fit=lambda *a: fitted.append(a))
    with pytest.raises(_error("IncompatibleAcquisitionFunctionError")):
        qNIPV().scorer(surrogate, space, _objective("pareto"), None)
    hybrid = _space(10)
    hybrid.type = SimpleNamespace(name="HYBRID")
    with pytest.raises(_error("IncompatibleAcquisitionFunctionError")):
        qNIPV().scorer(surrogate, hybrid, _objective(), None)
    Affine = type("AffineTransformation", (), {})
    incompat = (NotImplementedError,)
    try:
        from baybe.exceptions import IncompatibilityError

        incompat = (IncompatibilityError,)
    except ImportError:
        pass
    with pytest.raises(incompat, match="does not support any target transformations"):
        qNIPV().scorer(surrogate, space, _objective(transformation=Affine()), None)
    with pytest.raises(incompat):
        qNIPV().scorer(surrogate, space, _objective("desirability"), None)
    assert not fitted
    with pytest.raises(IncompatibleAcquisitionFunctionError):
        qNIPV().to_engine(None, space, _objective(), None)


def _fake_model(wide: bool = False, n: int = 64):
    m = _lib.Model()
    m.abi_version = _lib.ABI_VERSION
    m.n = m.n_pad = n
    m.n_chunks = 1
    m.d = m.d_pad = 2048 if wide else 20
    m.family = _lib.KERNEL_FAMILY["rbf"]
    m.task_col = -1
    m.n_tasks = 1
    m.y_std = m.prior_scale = m.r_scale = 1.0
    m.wide = int(wide)
    for name, ctype in _lib.Model._fields_:
        if name.startswith("d_") and ctype is C.c_void_p:
            setattr(m, name, 1 << 20)
    return m


@pytest.mark.parametrize("case", ["n_cond 32", "wide", "n 300", "null key", "bad noise", "no workspace", "M 0",
                                  "N 0"])
def test_nipv_score_checks_before_any_cuda_call(case):
    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    from baybe_b200.build import build

    build(verbose=False)
    lib = _lib.load()
    m = _fake_model(wide=case == "wide", n=300 if case == "n 300" else 64)
    p = C.c_void_p(1 << 20)
    noise = (C.c_float * 1)(-1.0 if case == "bad noise" else 0.01)
    N = 0 if case == "N 0" else 100
    M = 0 if case == "M 0" else 50
    n_cond = 32 if case == "n_cond 32" else 0
    key = None if case == "null key" else p
    ws_bytes = 16 if case == "no workspace" else 1 << 30
    rc = lib.bb_nipv_score(C.byref(m), noise, 1.0, p, N, p, M, p, n_cond, p, p, p, None, None, key, 0, p, ws_bytes,
                           None)
    expected = {"n_cond 32": _lib.BB_ERR_INVALID, "wide": _lib.BB_ERR_UNSUPPORTED, "n 300": _lib.BB_ERR_UNSUPPORTED,
                "null key": _lib.BB_ERR_INVALID, "bad noise": _lib.BB_ERR_INVALID,
                "no workspace": _lib.BB_ERR_WORKSPACE, "M 0": _lib.BB_ERR_INVALID, "N 0": 0}[case]
    assert rc == expected, lib.bb_last_error()
    if case == "n 300":
        assert b"at most 256" in lib.bb_last_error()


# ---- scorer algebra on a float64 stand-in engine ------------------------------------------------------------------------
@pytest.fixture()
def f64_engine(monkeypatch):
    from baybe_b200 import nipv
    from tests import nipv_oracle as po

    monkeypatch.setattr(nipv, "_joint_posterior", po.joint_posterior_f64)
    monkeypatch.setattr(nipv, "_nipv_score", po.nipv_score_f64)


def _setup(n=20, N=60, M=25, seed=0, task=False):
    import dataclasses

    from baybe_b200.nipv import NipvScorer
    from baybe_b200.synthetic import numeric_grid_workload, task_workload
    from tests.nipv_oracle import NipvStandInGP

    if task:
        w = task_workload(N_per_task=40, n_tasks=2, d_num=3, n_per_task=10, seed=seed)
        w = dataclasses.replace(w, noise=np.array([2e-2, 5e-2]))
    else:
        w = dataclasses.replace(numeric_grid_workload(N=300, d=4, n=n, seed=seed), noise=np.array([2e-2]))
    gp = NipvStandInGP(**w.gp_kwargs())
    rng = np.random.default_rng(seed)
    f32 = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731  the scorer sends fp32 rows
    x = f32(w.candidates[rng.choice(len(w.candidates), N, replace=False)])
    xm = f32(w.candidates[rng.choice(len(w.candidates), M, replace=False)])
    return w, gp, NipvScorer(gp, AcqConfig("qNIPV"), xm), x, xm


@pytest.mark.parametrize("P,Q,task", [(0, 0, False), (3, 0, False), (2, 2, False), (0, 3, False), (2, 1, True)])
def test_values_equal_the_definition(f64_engine, P, Q, task):
    from tests.nipv_oracle import nipv_definition

    w, gp, sc, x, xm = _setup(task=task)
    rng = np.random.default_rng(5)
    other = w.candidates[rng.choice(len(w.candidates), P + Q, replace=False)]
    pend, batch = (other[:P] if P else None), (other[P:] if Q else None)
    got = sc.scores(x, pend, seed=0, n_samples=64, batch=batch)
    ref = nipv_definition(gp, x, xm, other)
    assert np.abs(got - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max())
    assert (got < 0).all()


def test_joint_value_matches_brute_force(f64_engine):
    from tests.nipv_oracle import batch_definition

    w, gp, sc, x, xm = _setup()
    pend = w.candidates[[3, 7]]
    for q in (1, 2, 4):
        rows = x[:q]
        got = sc.joint_value(rows, pend, seed=0, n_samples=64)
        ref = batch_definition(gp, np.concatenate([rows, pend]), xm)
        assert abs(got - ref) <= 1e-10 * max(1.0, abs(ref))


def test_greedy_batch_matches_brute_force(f64_engine):
    from baybe_b200.recommenders import greedy_select
    from tests.nipv_oracle import nipv_definition

    w, gp, sc, x, xm = _setup(N=40)
    chosen, vals = greedy_select(sc, sc.cfg, torch.from_numpy(x), x.shape[1], 3, None, seed=1, n_samples=64)
    assert len(set(chosen)) == 3
    for r in range(3):  # a round reports its winner's value from the packed key, whose IVR is float32
        ref = nipv_definition(gp, x, xm, x[chosen[:r]])
        assert abs(ref[chosen[r]] - vals[r]) <= 1e-6 * max(1.0, abs(vals[r]))
        ref[chosen[:r]] = -np.inf
        assert ref[chosen[r]] >= ref.max() - 1e-6 * abs(ref.max())


def test_more_than_31_conditioning_points_raise(f64_engine):
    w, gp, sc, x, xm = _setup(n=40)
    with pytest.raises(NotImplementedError, match="at most 31"):
        sc.scores(x[:2], w.candidates[:32], seed=0, n_samples=64)


# ---- Campaign glue on the float64 stand-in engine -----------------------------------------------------------------------
@pytest.fixture()
def bb(monkeypatch, f64_engine):
    ref_dir = ROOT / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe_b200 import baybe_plugin, surrogates
    from tests.nipv_oracle import NipvStandInGP

    monkeypatch.setattr(surrogates, "DeviceGP", NipvStandInGP)
    return baybe_plugin


def test_nipv_campaign_on_the_stand_in_engine(bb):
    from baybe.acquisition import acqfs

    from baybe_b200.nipv import NipvScorer
    from tests.test_nei import check_noisy_flow, noisy_campaign

    camp, space = noisy_campaign(bb, acqfs.qNegIntegratedPosteriorVariance())
    vals = check_noisy_flow(camp, space, np.random.default_rng(0), tol=1e-6)
    assert isinstance(camp.recommender._scorer, NipvScorer) and camp.recommender._scorer.M == len(space.discrete.exp_rep)
    assert (vals < 0).all()


def test_fps_integration_points_come_from_baybe_everywhere(bb, monkeypatch):
    from baybe.acquisition import acqfs

    from baybe_b200 import nipv
    from tests.test_mo import measure
    from tests.test_nei import noisy_campaign

    acqf = acqfs.qNegIntegratedPosteriorVariance(sampling_n_points=17, sampling_method="FPS")
    camp, space = noisy_campaign(bb, acqf)
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=1), np.random.default_rng(0),
                                  ("yield",)))
    seen = []
    init = nipv.NipvScorer.__init__

    def spy(self, gp, cfg, integration):
        seen.append(np.asarray(integration, dtype=np.float64))
        init(self, gp, cfg, integration)

    monkeypatch.setattr(nipv.NipvScorer, "__init__", spy)
    assert len(camp.recommend(batch_size=2)) == 2
    vals = camp.acquisition_values(space.discrete.exp_rep.head(15))
    jv = camp.joint_acquisition_value(space.discrete.exp_rep.head(2))
    assert np.isfinite(vals.to_numpy()).all() and np.isfinite(jv)
    ref = acqf.get_integration_points(space).to_numpy(dtype=np.float64)
    assert len(seen) == 3 and all(s.shape == ref.shape for s in seen)


def test_minimized_target_recommends_the_same_rows(bb):
    from baybe.acquisition import acqfs
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget

    from tests.test_mo import measure
    from tests.test_nei import noisy_campaign

    out = []
    for minimize in (False, True):
        camp, space = noisy_campaign(bb, acqfs.qNegIntegratedPosteriorVariance(),
                                     SingleTargetObjective(NumericalTarget("yield", minimize=minimize)))
        camp.add_measurements(measure(space.discrete.exp_rep.sample(12, random_state=1), np.random.default_rng(0),
                                      ("yield",)))
        out.append((list(camp.recommend(batch_size=3).index), camp.acquisition_values(space.discrete.exp_rep.head(30))))
    assert out[0][0] == out[1][0]
    assert np.allclose(out[0][1].to_numpy(), out[1][1].to_numpy(), rtol=1e-9, atol=0.0)


def test_nipv_subset_constraint_on_the_stand_in_engine(bb):
    from baybe import Campaign
    from baybe.acquisition import acqfs
    from baybe.constraints import DiscreteBatchConstraint
    from baybe.objectives import SingleTargetObjective
    from baybe.parameters import CategoricalParameter, NumericalDiscreteParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    params = [NumericalDiscreteParameter("x", values=[0.0, 0.25, 0.5, 0.75, 1.0]),
              NumericalDiscreteParameter("y", values=[0.0, 0.5, 1.0]),
              CategoricalParameter("cat", values=["p", "q", "r"], encoding="OHE")]
    space = SearchSpace.from_product(params, constraints=[DiscreteBatchConstraint(parameters=["cat"])])
    hp = {"lengthscale": np.full(len(space.comp_rep_columns), 0.7), "noise": 5e-2, "mean_const": 0.0}
    rec = bb.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp),
                                    acquisition_function=acqfs.qNegIntegratedPosteriorVariance())
    camp = Campaign(space, SingleTargetObjective(NumericalTarget("t1")), rec)
    rows = space.discrete.exp_rep.sample(8, random_state=0)
    meas = rows.copy()
    meas["t1"] = rows["x"] - (rows["y"] - 0.5) ** 2 + np.random.default_rng(5).normal(0, 0.05, len(rows))
    camp.add_measurements(meas)
    batch = camp.recommend(batch_size=3)
    assert len(batch) == 3 and batch["cat"].nunique() == 1


def test_nipv_rejections_through_the_campaign(bb):
    from baybe import Campaign
    from baybe.acquisition import acqfs
    from baybe.exceptions import IncompatibilityError
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget
    from baybe.transformations import AffineTransformation

    from tests.test_mo import measure
    from tests.test_nei import noisy_campaign

    camp, space = noisy_campaign(bb, acqfs.qNegIntegratedPosteriorVariance(),
                                 SingleTargetObjective(NumericalTarget("yield",
                                                                       transformation=AffineTransformation(2.0, 1.0))))
    assert isinstance(camp, Campaign)
    camp.add_measurements(measure(space.discrete.exp_rep.sample(8, random_state=1), np.random.default_rng(0),
                                  ("yield",)))
    with pytest.raises(IncompatibilityError, match="does not support any target transformations"):
        camp.recommend(batch_size=1)
