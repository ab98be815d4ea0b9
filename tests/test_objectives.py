"""CPU tests of objectives that are not affine in their targets (desirability, non-affine single targets): the
compiled programs against the reference's own transformations, the scalarisers, the sampling recipe against
quadrature, the argument checks of ``bb_objective_score`` and the Campaign glue on a float64 stand-in engine."""
from __future__ import annotations

import ctypes as C
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import objectives as ob
from tests import objective_oracle as oo

ROOT = Path(__file__).resolve().parents[1]


def _reference():
    ref_dir = ROOT / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401


# ---- program semantics --------------------------------------------------------------------------------------------
def _transformations():
    from baybe.transformations import (AbsoluteTransformation, AffineTransformation, BellTransformation,
                                       ClampingTransformation, ExponentialTransformation, IdentityTransformation,
                                       LogarithmicTransformation, PowerTransformation, SigmoidTransformation,
                                       TriangularTransformation, TwoSidedAffineTransformation)
    from baybe.transformations.composite import (AdditiveTransformation, ChainedTransformation,
                                                 MultiplicativeTransformation)

    return {
        "identity": IdentityTransformation(),
        "affine": AffineTransformation(factor=-2.5, shift=0.3),
        "affine factor 0": AffineTransformation(factor=0.0, shift=1.5),
        "clamp both": ClampingTransformation(min=-1.0, max=2.0),
        "clamp lower": ClampingTransformation(min=0.5),
        "clamp upper": ClampingTransformation(max=0.5),
        "two-sided": TwoSidedAffineTransformation(slope_left=-0.5, slope_right=2.0, midpoint=0.7),
        "two-sided zero slope": TwoSidedAffineTransformation(slope_left=0.0, slope_right=1.0, midpoint=0.0),
        "bell": BellTransformation(center=0.4, sigma=0.8),
        "absolute": AbsoluteTransformation(),
        "triangular": TriangularTransformation.from_margins(peak=1.0, margins=(0.5, 2.0)),
        "log": LogarithmicTransformation(),
        "exp": ExponentialTransformation(),
        "power even": PowerTransformation(exponent=2),
        "power odd": PowerTransformation(exponent=3),
        "sigmoid": SigmoidTransformation(center=0.2, steepness=-3.0),
        "chained": ChainedTransformation([AffineTransformation(2.0, 1.0), BellTransformation(0.0, 2.0),
                                          AffineTransformation(3.0, -1.0)]),
        "additive": AdditiveTransformation([BellTransformation(0.0, 1.0), AbsoluteTransformation()]),
        "multiplicative": MultiplicativeTransformation([ExponentialTransformation(),
                                                        SigmoidTransformation(center=1.0, steepness=2.0)]),
        "nested": ChainedTransformation([AffineTransformation(0.5, 0.1), AdditiveTransformation([
            MultiplicativeTransformation([AbsoluteTransformation(), BellTransformation(0.0, 1.5)]),
            SigmoidTransformation(center=0.5, steepness=1.5)]), ExponentialTransformation()]),
    }


def _targets():
    from baybe.targets import NumericalTarget

    return {
        "match_triangular": NumericalTarget.match_triangular("t", cutoffs=(-1.0, 3.0)),
        "match_bell": NumericalTarget.match_bell("t", match_value=0.5, sigma=1.2),
        "match_absolute": NumericalTarget.match_absolute("t", match_value=0.3),
        "normalized_ramp": NumericalTarget.normalized_ramp("t", cutoffs=(-1.0, 2.0)),
        "normalized_ramp desc": NumericalTarget.normalized_ramp("t", cutoffs=(-1.0, 2.0), descending=True),
        "normalized_sigmoid": NumericalTarget.normalized_sigmoid("t", anchors=[(-1.0, 0.1), (1.0, 0.9)]),
        "clamp normalize": NumericalTarget("t").clamp(-2.0, 3.0).normalize(),
        "log": NumericalTarget("t").log(),
        "exp": NumericalTarget("t").exp(),
        "power": NumericalTarget("t").power(3),
        "minimised exp": NumericalTarget("t", minimize=True).exp(),
    }


def _grid():
    y = torch.linspace(-4.0, 4.0, 801, dtype=torch.float64)
    return torch.cat([y, torch.tensor([0.0, 1e-300, -1e-300, 700.0, 709.0, 710.0, -745.0])])


def _same(a: torch.Tensor, b: torch.Tensor):
    a, b = a.double(), b.double()
    assert torch.equal(torch.isnan(a), torch.isnan(b))
    ok = ~torch.isnan(a)
    assert torch.equal(torch.isinf(a[ok]), torch.isinf(b[ok]))
    fin = ok & ~torch.isinf(a)
    assert torch.allclose(a[fin], b[fin], rtol=1e-12, atol=1e-12)


def test_programs_equal_the_reference_transformations():
    _reference()
    y = _grid()
    for name, tr in _transformations().items():
        prog = ob.program_of(tr, name)
        ref = tr(y.clone())
        _same(oo.run_program(prog, y), ref)
        _same(torch.from_numpy(ob.evaluate_program(prog, y.numpy())), ref)  # the product's host evaluator


def test_target_factories_and_orientation_equal_the_reference():
    _reference()
    from baybe.objectives import DesirabilityObjective, SingleTargetObjective
    from baybe.targets import NumericalTarget

    y = _grid()
    for name, t in _targets().items():
        obj = SingleTargetObjective(t)
        comp = ob.compile_objective(obj)
        oriented = obj._oriented_targets[0].transformation
        _same(oo.run_program(comp.programs[0], y), oriented(y.clone()))
    # desirability: minimised targets become 1 - y (negate + 1) before their transformation's image
    t1 = NumericalTarget.normalized_ramp("a", cutoffs=(0.0, 1.0))
    t2 = NumericalTarget.normalized_ramp("b", cutoffs=(0.0, 2.0), descending=False)
    t2 = NumericalTarget("b", transformation=t2.transformation, minimize=True)
    d = DesirabilityObjective([t1, t2], weights=[1.0, 3.0], require_normalization=False)
    comp = ob.compile_objective(d)
    for m, t in enumerate(d._oriented_targets):
        _same(oo.run_program(comp.programs[m], y), t.transformation(y.clone()))
    assert np.allclose(comp.weights, [0.25, 0.75])
    # minimised single target: plain negation
    s = SingleTargetObjective(NumericalTarget("c", minimize=True).exp())
    _same(oo.run_program(ob.compile_objective(s).programs[0], y), -torch.exp(y))


def test_scalarizers_equal_the_reference():
    _reference()
    from baybe.objectives.desirability import _geometric_mean

    rng = np.random.default_rng(0)
    T = torch.from_numpy(rng.random((50, 3)))
    T[:5, 1] = 0.0  # zero desirabilities take the eps path
    w = torch.tensor([1.0, 2.0, 5.0]) / 8.0
    ref = _geometric_mean(T, torch.tensor([1.0, 2.0, 5.0], dtype=torch.float64))
    _same(oo.scalarize(T, "GEOM_MEAN", w.numpy()), ref)
    _same(torch.from_numpy(ob.scalarize(T.numpy(), "GEOM_MEAN", w.numpy())), ref)
    _same(torch.from_numpy(ob.scalarize(T.numpy(), "MEAN", w.numpy())), T @ w.double())


# ---- sampling recipe against quadrature -------------------------------------------------------------------------------
def test_mc_qei_of_a_bell_target_matches_quadrature():
    from scipy import integrate
    from scipy.stats import norm

    from baybe_b200 import _lib

    prog = [("BELL", (0.3, 0.7, 0.0))]
    mu, sd, best_f = 0.1, 0.9, 0.6
    S = 4096
    z = oracle.sobol_normal_samples(S, 1, seed=7)
    ops = [_lib.OBJ_OP[o] for o, _ in prog]
    args = [v for _, a in prog for v in a]
    params = [1.0, best_f, 0.2, 1.0, 0.0, 1e-6, 1e-2, 1e-3]
    val, _ = oo.objective_score_f64(torch.tensor([[mu]]), torch.tensor([[sd * sd]]), None, None, None, None, z, None,
                                    _lib.ACQ_KIND["qEI"], params, 0, ops, args, [1], [1.0], 0, True)
    f = lambda y: max(math.exp(-((y - 0.3) / 0.7) ** 2 / 2) - best_f, 0.0) * norm.pdf(y, mu, sd)  # noqa: E731
    exact, _ = integrate.quad(f, mu - 12 * sd, mu + 12 * sd, points=[0.3], limit=200)
    vals = np.maximum(np.exp(-(((mu + sd * z[:, 0].numpy()) - 0.3) / 0.7) ** 2 / 2) - best_f, 0.0)
    mc_err = 4.0 * vals.std() / math.sqrt(S)  # 4 standard errors of plain MC; scrambled Sobol does better
    assert abs(float(val[0]) - exact) < mc_err, (float(val[0]), exact, mc_err)


# ---- bb_objective_score argument checks -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _call(lib, **over):
    from baybe_b200 import _lib
    from baybe_b200.engine import objective_struct

    a = _lib.AcqSpec(kind=over.pop("kind", _lib.ACQ_KIND["qLogEI"]), tau_relu=over.pop("tau_relu", 1e-6),
                     tau_max=1e-2, tau_pi=1e-3)
    M = over.pop("M", 2)
    progs = over.pop("progs", [[(_lib.OBJ_OP["BELL"], (0.0, 1.0, 0.0))]] * M)
    obj = objective_struct(min(M, 8), over.pop("scal", 2 if M > 1 else 0), progs[:8], [1.0 / max(M, 1)] * min(M, 8))
    obj.n_targets = M
    for k, v in over.pop("raw", {}).items():
        setattr(obj, k, v)
    p = C.c_void_p(1 << 20)
    args = dict(a=None if over.pop("null_acq", False) else C.byref(a),
                obj=None if over.pop("null_obj", False) else C.byref(obj), N=100, mu=p, var=p, P=0, cross=None,
                linv=None, w=None, pend=None, z=p, S=64, keep=None, score=p, key=p, offset=0, stream=None)
    args.update(over)
    return lib.bb_objective_score(*args.values())


def _ops(*names):
    from baybe_b200 import _lib

    return [(_lib.OBJ_OP[n], (2.0, 0.0, 0.0)) for n in names]


_BAD = [
    ("null spec", dict(null_acq=True), "invalid", b"spec is null"),
    ("null objective", dict(null_obj=True), "invalid", b"objective is null"),
    ("kind qEHVI", dict(kind=11), "invalid", b"not a single-objective"),
    ("tau_relu 0", dict(tau_relu=0.0), "invalid", b"tau_relu"),
    ("M = 0", dict(M=0, progs=[]), "unsupported", b"n_targets=0"),
    ("M = 9", dict(M=9, progs=[[]] * 9), "unsupported", b"n_targets=9"),
    ("NONE with two targets", dict(scal=0), "invalid", b"scalarizer NONE"),
    ("unknown scalarizer", dict(scal=7), "invalid", b"unknown scalarizer"),
    ("33 ops", dict(raw={"n_ops": (C.c_int32 * 8)(33, 1)}), "unsupported", b"33 ops"),
    ("unknown opcode", dict(progs=[[(12, (0.0, 0.0, 0.0))], []]), "invalid", b"unknown opcode 12"),
    ("stack depth 5", dict(progs=[_ops("DUP_INPUT", "DUP_INPUT", "DUP_INPUT", "DUP_INPUT"), []]), "unsupported",
     b"stack depth 5"),
    ("pop of an empty stack", dict(progs=[_ops("ADD"), []]), "invalid", b"pops an empty stack"),
    ("two entries left", dict(progs=[_ops("DUP_INPUT"), []]), "invalid", b"leaves 2 stack entries"),
    ("non-integer power", dict(progs=[[(7, (2.5, 0.0, 0.0))], []]), "unsupported", b"non-integer power"),
    ("analytic GEOM_MEAN", dict(kind=6), "unsupported", b"MEAN scalarisation"),
    ("analytic non-affine", dict(kind=6, scal=1), "unsupported", b"affine targets"),
    ("S = 0", dict(S=0), "invalid", b"S=0"),
    ("S = 1025", dict(S=1025), "invalid", b"S=1025"),
    ("P = 32", dict(P=32), "invalid", b"n_pending=32"),
    ("null key", dict(key=None), "invalid", b"null best key"),
    ("null mu", dict(mu=None), "invalid", b"null buffer"),
    ("pending without terms", dict(P=2, cross=C.c_void_p(1 << 20), linv=C.c_void_p(1 << 20), w=C.c_void_p(1 << 20)),
     "invalid", b"pending terms"),
    ("negative offset", dict(offset=-1), "invalid", b"32-bit key"),
]


@pytest.mark.parametrize("case,over,status,msg", _BAD, ids=[c for c, *_ in _BAD])
def test_bb_objective_score_rejects_bad_arguments_before_any_cuda_call(lib, case, over, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    rc = _call(lib, **over)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


def test_bb_objective_score_accepts_an_empty_candidate_set(lib):
    assert _call(lib, N=0, mu=None, var=None) == 0


# ---- Campaign glue on a float64 stand-in engine -------------------------------------------------------------------------
@pytest.fixture()
def bb(monkeypatch):
    """The stand-in engine of tests/test_mo.py's ``bb`` fixture, with ``bb_objective_score`` replaced by its float64
    definition."""
    _reference()
    from baybe_b200 import baybe_plugin, surrogates
    from tests.helpers import OracleBackedGP

    class StandInGP(OracleBackedGP):
        def pending_stats(self, pending):
            p = np.asarray(pending, dtype=np.float64).reshape(-1, self.d)
            mu, cov = oracle.posterior_joint(self.om, p)
            return p, None, mu.float(), cov.float()

        def cross_covariance(self, x, pend_x, beta):
            x = np.asarray(x, dtype=np.float64)
            mu, var = oracle.posterior(self.om, x)
            P = len(pend_x)
            _, cov = oracle.posterior_joint(self.om, np.concatenate([pend_x, x]))
            return mu.float(), var.float(), cov[P:, :P].float().contiguous()

    monkeypatch.setattr(surrogates, "DeviceGP", StandInGP)
    monkeypatch.setattr(ob, "_objective_score", oo.objective_score_f64)
    return baybe_plugin


def desirability_campaign(plugin, acqf=None, scalarizer="GEOM_MEAN", targets=None, hp=True, **kw):
    """Shared by the CPU and GPU Campaign tests: the 216-row space of tests/test_mo.py, yield and cost normalised
    by clamps (cost minimised)."""
    from baybe import Campaign
    from baybe.objectives import DesirabilityObjective
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate
    from tests.test_mo import pareto_campaign

    _, space = pareto_campaign(plugin, None)
    d = len(space.comp_rep_columns)
    hyper = {"lengthscale": np.full(d, 0.9), "noise": 5e-3, "mean_const": 0.0} if hp else None
    targets = targets or [NumericalTarget("yield").clamp(45.0, 60.0).normalize(),
                          NumericalTarget("cost", minimize=True).clamp(4.0, 7.0).normalize()]
    obj = DesirabilityObjective(targets, scalarizer=scalarizer, **kw)
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hyper),
                                        n_mc_samples=128, **({} if acqf is None else {"acquisition_function": acqf}))
    return Campaign(space, obj, rec, allow_recommending_already_measured=False), space


def check_flow(camp, space, rng, batch=3, tol=1e-4):
    """Recommendation = arg-max of acquisition_values, single-row joint value = own value, pending honoured."""
    from tests.test_mo import measure

    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, rng))
    rec = camp.recommend(batch_size=batch)
    assert len(rec) == batch and rec.index.is_unique and not set(rec.index) & set(seed_rows.index)
    camp.add_measurements(measure(rec, rng))
    torch.manual_seed(11)
    r1 = camp.recommend(batch_size=1)
    torch.manual_seed(11)
    vals = camp.acquisition_values(space.discrete.exp_rep)
    remaining = vals.drop(index=list(seed_rows.index) + list(rec.index))
    assert float(vals.loc[r1.index[0]]) >= float(remaining.max()) - tol * max(1.0, abs(float(remaining.max())))
    torch.manual_seed(11)
    jv = camp.joint_acquisition_value(r1)
    assert abs(jv - float(vals.loc[r1.index[0]])) <= tol * max(1.0, abs(jv))
    rec3 = camp.recommend(batch_size=3, pending_experiments=r1)
    assert len(rec3) == 3 and r1.index[0] not in rec3.index
    return vals


def test_geometric_desirability_campaign_on_the_stand_in_engine(bb):
    camp, space = desirability_campaign(bb)
    vals = check_flow(camp, space, np.random.default_rng(0), tol=0.0)
    assert np.isfinite(vals.to_numpy()).all()


def test_desirability_subset_constraint_on_the_stand_in_engine(bb, monkeypatch):
    from baybe import Campaign
    from baybe.constraints import DiscreteBatchConstraint
    from baybe.objectives import DesirabilityObjective
    from baybe.parameters import CategoricalParameter, NumericalDiscreteParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    params = [NumericalDiscreteParameter("x", values=[0.0, 0.25, 0.5, 0.75, 1.0]),
              NumericalDiscreteParameter("y", values=[0.0, 0.5, 1.0]),
              CategoricalParameter("cat", values=["p", "q", "r"], encoding="OHE")]
    space = SearchSpace.from_product(params, constraints=[DiscreteBatchConstraint(parameters=["cat"])])
    hp = {"lengthscale": np.full(len(space.comp_rep_columns), 0.7), "noise": 1e-2, "mean_const": 0.0}
    rec = bb.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp), n_mc_samples=128)
    obj = DesirabilityObjective([NumericalTarget("t1").clamp(-1.0, 1.5).normalize(),
                                 NumericalTarget.match_bell("t2", match_value=0.5, sigma=0.5)])
    camp = Campaign(space, obj, rec)
    rows = space.discrete.exp_rep.sample(8, random_state=0)
    meas = rows.copy()
    rng = np.random.default_rng(5)
    shift = rows["cat"].map({"p": 0.0, "q": 0.3, "r": -0.2}).astype(float)
    meas["t1"] = rows["x"] - (rows["y"] - 0.5) ** 2 + shift + rng.normal(0, 0.02, len(rows))
    meas["t2"] = rows["x"] ** 2 + rows["y"] - shift + rng.normal(0, 0.02, len(rows))
    camp.add_measurements(meas)
    batches, values = [], []
    without = bb.B200BotorchRecommender._recommend_discrete_without_subsets
    call = bb.EngineAcquisitionFunction.__call__

    def spy_batch(self, *args):
        idx = without(self, *args)
        batches.append(list(idx))
        return idx

    def spy_value(self, X):
        out = call(self, X)
        values.append(float(out[0]))
        return out

    monkeypatch.setattr(bb.B200BotorchRecommender, "_recommend_discrete_without_subsets", spy_batch)
    monkeypatch.setattr(bb.EngineAcquisitionFunction, "__call__", spy_value)
    batch = camp.recommend(batch_size=3)
    assert len(batch) == 3 and batch["cat"].nunique() == 1
    assert len(batches) == len(values) >= 2
    assert list(batch.index) == batches[int(np.argmax(values))]


def test_partial_measurements_under_desirability(bb):
    from tests.test_mo import measure

    camp, space = desirability_campaign(bb)
    rows = measure(space.discrete.exp_rep.sample(14, random_state=3), np.random.default_rng(2))
    rows.loc[rows.index[:3], "cost"] = np.nan
    rows.loc[rows.index[3:5], "yield"] = np.nan
    camp.add_measurements(rows)
    rec = camp.recommend(batch_size=2)
    assert len(rec) == 2 and not set(rec.index) & set(rows.index)


@pytest.mark.parametrize("acqf", ["qEI", "qUCB"])
def test_match_bell_single_target(bb, acqf):
    from baybe import Campaign
    from baybe.acquisition import qExpectedImprovement, qUpperConfidenceBound
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate
    from tests.test_mo import pareto_campaign

    _, space = pareto_campaign(bb, None)
    hp = {"lengthscale": np.full(len(space.comp_rep_columns), 0.9), "noise": 5e-3, "mean_const": 0.0}
    a = {"qEI": qExpectedImprovement(), "qUCB": qUpperConfidenceBound(beta=0.5)}[acqf]
    rec = bb.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp),
                                    acquisition_function=a, n_mc_samples=128)
    camp = Campaign(space, SingleTargetObjective(NumericalTarget.match_bell("yield", match_value=55.0, sigma=2.0)),
                    rec, allow_recommending_already_measured=False)
    from tests.test_mo import measure

    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, np.random.default_rng(0), ("yield",)))
    torch.manual_seed(3)
    r1 = camp.recommend(batch_size=1)
    torch.manual_seed(3)
    vals = camp.acquisition_values(space.discrete.exp_rep).drop(index=seed_rows.index)
    assert r1.index[0] == vals.idxmax()
    assert len(camp.recommend(batch_size=3)) == 3


def test_mean_desirability_with_analytic_ei_and_the_best_f_quirk(bb):
    from baybe.acquisition import ExpectedImprovement
    from baybe.targets import NumericalTarget

    from tests.test_mo import measure

    targets = [NumericalTarget("yield"), NumericalTarget("cost", minimize=True)]
    camp, space = desirability_campaign(bb, ExpectedImprovement(), scalarizer="MEAN", targets=targets,
                                        require_normalization=False, weights=[1.0, 3.0])
    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, np.random.default_rng(0)))
    vals = camp.acquisition_values(space.discrete.exp_rep)
    r1 = camp.recommend(batch_size=1)
    assert r1.index[0] == vals.drop(index=seed_rows.index).idxmax()
    # the value by hand: posterior transform without the + 1, best_f with it (higher by the minimised weight 0.75)
    surrogate = camp.recommender.get_surrogate(space, camp.objective, camp.measurements)
    from baybe.objectives import DesirabilityObjective

    stats = surrogate.posterior_stats(space.discrete.exp_rep, stats=("mean", "var"))
    mean = 0.25 * stats["yield_mean"] - 0.75 * stats["cost_mean"]
    sd = np.sqrt(0.25 ** 2 * stats["yield_var"] + 0.75 ** 2 * stats["cost_var"])
    tr = stats.loc[seed_rows.index]
    best_f = float((0.25 * tr["yield_mean"] + 0.75 * (1.0 - tr["cost_mean"])).max())
    from scipy.stats import norm

    u = (mean - best_f) / sd
    ei = sd * (norm.pdf(u) + u * norm.cdf(u))
    assert np.allclose(vals.to_numpy(), ei.to_numpy(), rtol=1e-5, atol=1e-9)
    assert isinstance(camp.objective, DesirabilityObjective)


def test_desirability_as_pre_transformation(bb):
    camp, space = desirability_campaign(bb, as_pre_transformation=True)
    from tests.test_mo import measure

    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    meas = measure(seed_rows, np.random.default_rng(0))
    camp.add_measurements(meas)
    rec = camp.recommend(batch_size=2)
    assert len(rec) == 2 and not set(rec.index) & set(seed_rows.index)
    surrogate = camp.recommender._surrogate_model
    assert surrogate._target_name == "Desirability"
    comp = ob.compile_objective(camp.objective)
    want = ob.evaluate_objective(comp, meas[["yield", "cost"]].to_numpy())
    got = surrogate.posterior_stats(seed_rows)["Desirability_mean"].to_numpy()
    assert np.allclose(got, want, atol=0.05)


# ---- rejections -------------------------------------------------------------------------------------------------------
def test_rejections(bb):
    from baybe.acquisition import ExpectedImprovement, UpperConfidenceBound
    from baybe.exceptions import IncompatibilityError
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget
    from baybe.transformations import CustomTransformation, PowerTransformation
    from baybe.transformations.composite import ChainedTransformation
    from baybe.transformations import AffineTransformation, BellTransformation

    from tests.test_mo import measure

    rng = np.random.default_rng(1)
    camp, space = desirability_campaign(bb, ExpectedImprovement())  # GEOM_MEAN
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng))
    with pytest.raises(IncompatibilityError):
        camp.recommend(batch_size=1)
    camp, space = desirability_campaign(bb, UpperConfidenceBound(), scalarizer="MEAN")  # non-affine targets
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng))
    with pytest.raises(IncompatibilityError):
        camp.recommend(batch_size=1)
    with pytest.raises(NotImplementedError, match="CustomTransformation"):
        ob.compile_objective(SingleTargetObjective(NumericalTarget("t", transformation=CustomTransformation(
            lambda x: x * 2))))
    with pytest.raises(NotImplementedError, match="non-integer"):
        ob.compile_objective(SingleTargetObjective(NumericalTarget("t", transformation=PowerTransformation(2.5))))
    from baybe.objectives import DesirabilityObjective

    nine = DesirabilityObjective([NumericalTarget(f"t{i}").clamp(0.0, 1.0) for i in range(9)])
    with pytest.raises(NotImplementedError, match="9 targets"):
        ob.compile_objective(nine)
    long = ChainedTransformation([t for i in range(20) for t in (BellTransformation(0.1 * i, 1.0),
                                                                 AffineTransformation(1.0 + i, 0.5))])
    with pytest.raises(NotImplementedError, match="ops"):
        ob.compile_objective(SingleTargetObjective(NumericalTarget("t", transformation=long)))
