"""CPU tests of the gradient path's host side (baybe_b200/continuous.py, the plugin's continuous and hybrid hooks) on a
float64 stand-in engine (tests/continuous_oracle.py: value and gradient by autograd of the oracle), and the argument
checks of ``bb_acq_grad`` before any CUDA call."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pandas as pd
import pytest
import torch

from baybe_b200.acquisition import AcqConfig
from baybe_b200.continuous import initial_starts, recommend_continuous_hybrid
from tests.continuous_oracle import OracleGradGP

ROOT = Path(__file__).resolve().parents[1]
REF = ROOT / "oracle" / "_ref" if (ROOT / "oracle" / "_ref" / "baybe").is_dir() else None
needs_ref = pytest.mark.skipif(REF is None, reason="the reference package (baybe) is not installed under oracle/_ref")


def _model(d=3, n=12, seed=0, family="matern52"):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 1, (n, d))
    y = np.sin(3 * X).sum(1) + 0.05 * rng.normal(size=n)
    ls = np.full(d, 0.4)
    return OracleGradGP(X, y, np.array([np.zeros(d), np.ones(d)]), family, ls, 1e-3, outputscale=1.3)


def test_start_selection_is_botorchs_initialize_q_batch():
    vals = torch.from_numpy(np.random.default_rng(3).normal(size=200))
    got = initial_starts(vals, 10, seed=17)
    # literal restatement: Boltzmann weights exp(eta * standardised value), eta = 1, multinomial without replacement,
    # the best row forced into the last slot if it was not drawn
    gen = torch.Generator().manual_seed(17)
    Z = (vals - vals.mean()) / vals.std()
    want = torch.multinomial(torch.exp(Z), 10, replacement=False, generator=gen)
    if not bool((want == vals.argmax()).any()):
        want[-1] = vals.argmax()
    assert torch.equal(got, want)
    assert int(vals.argmax()) in got.tolist()
    assert torch.equal(initial_starts(vals[:5], 10, seed=1), torch.arange(5))


class _Spy:
    """Records the pending points of every value_and_grad call."""

    def __init__(self, gp):
        self.gp, self.pending_sizes, self.last_pending = gp, [], None

    def __getattr__(self, name):
        return getattr(self.gp, name)

    def value_and_grad(self, acq, x, z, pending=None):
        self.pending_sizes.append(0 if pending is None else len(pending))
        self.last_pending = None if pending is None else np.asarray(pending).copy()
        return self.gp.value_and_grad(acq, x, z, pending)


def test_hybrid_greedy_keeps_discrete_and_fixed_columns_and_passes_pending():
    gp = _model(d=4)
    spy = _Spy(gp)
    disc = np.array([[0.0], [0.5], [1.0]])
    cb = np.array([[0.0, 0.2, 0.1], [1.0, 0.6, 0.9]])
    acq = AcqConfig("qEI", best_f=gp.best_f(AcqConfig("qEI")))
    pend = np.array([[0.5, 0.3, 0.4, 0.5]])
    pts, idx, value = recommend_continuous_hybrid(spy, acq, disc, cb, 3, pend, n_samples=64, seed=5, n_raw_samples=16,
                                                  n_restarts=4, fixed={1: 0.45})
    assert pts.shape == (3, 4) and len(idx) == 3
    for r, k in zip(pts, idx):
        assert r[0] == disc[k, 0]               # the discrete column is one of the configurations, exactly
        assert r[2] == 0.45                     # the fixed parameter never moves
        assert np.all(r[1:] >= cb[0] - 1e-12) and np.all(r[1:] <= cb[1] + 1e-12)
    # greedy step j optimises given pending = [pending experiments; x_1 .. x_{j-1}]
    sizes = sorted(set(spy.pending_sizes))
    assert sizes == [1, 2, 3]
    np.testing.assert_array_equal(spy.last_pending, np.vstack([pend, pts[:2]]))
    want = float(gp.score_joint(acq, pts[:1], np.vstack([pts[1:], pend]),
                                __import__("baybe_b200.engine", fromlist=["x"]).sobol_normal_samples(64, 4, 5))[0])
    assert value == pytest.approx(want, rel=1e-6)


def test_continuous_polish_reaches_a_stationary_point_on_the_stand_in():
    gp = _model(d=2, n=10, seed=4)
    acq = AcqConfig("EI", best_f=gp.best_f(AcqConfig("EI")))
    cb = np.array([[0.0, 0.0], [1.0, 1.0]])
    pts, idx, value = recommend_continuous_hybrid(gp, acq, np.zeros((1, 0)), cb, 1, seed=2)
    assert idx == [0]
    g = gp.value_and_grad(acq, pts, None)[1].double().numpy()[0]
    on_bound = (np.abs(pts[0] - cb[0]) < 1e-9) | (np.abs(pts[0] - cb[1]) < 1e-9)
    assert np.all(np.abs(np.where(on_bound, 0.0, g)) <= 1e-3 * max(1.0, np.abs(g).max()))
    grid = np.stack(np.meshgrid(np.linspace(0, 1, 41), np.linspace(0, 1, 41)), -1).reshape(-1, 2)
    assert value >= float(gp.score(acq, grid, None)[0].max()) - 1e-6


def test_analytic_batch_and_task_model_are_rejected():
    gp = _model(d=2)
    cb = np.array([[0.0, 0.0], [1.0, 1.0]])
    with pytest.raises(ValueError, match="one point at a time"):
        recommend_continuous_hybrid(gp, AcqConfig("UCB"), np.zeros((1, 0)), cb, 2)
    gp.task_col = 1
    with pytest.raises(NotImplementedError, match="single-task"):
        recommend_continuous_hybrid(gp, AcqConfig("qEI"), np.zeros((1, 0)), cb, 1)


# ---- bb_acq_grad: argument checks before any CUDA call -------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _fake(wide=False, task=False, n_pad=64):
    from tests.test_abi import _fake_model

    m = _fake_model(wide, 1)
    m.n_pad = n_pad
    if task:
        m.task_col = 0
    return m


@pytest.mark.parametrize("case, status, msg", [
    ("null model", "invalid", b"model struct"),
    ("kind 11", "invalid", b"single-target"),
    ("wide", "unsupported", b"wide-feature"),
    ("task", "unsupported", b"task parameter"),
    ("n_pad 512", "unsupported", b"n_pad=512"),
    ("pending analytic", "invalid", b"Monte Carlo"),
    ("33 pending", "invalid", b"n_pending=33"),
    ("S 0", "invalid", b"S=0"),
    ("null samples", "invalid", b"base samples"),
    ("null pending", "invalid", b"pending buffer"),
    ("null output", "invalid", b"null buffer"),
])
def test_acq_grad_rejects_bad_arguments_before_any_cuda_call(lib, case, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    m = _fake(wide=case == "wide", task=case == "task", n_pad=512 if case == "n_pad 512" else 64)
    kind = {"kind 11": 11, "pending analytic": _lib.ACQ_KIND["EI"]}.get(case, _lib.ACQ_KIND["qEI"])
    a = _lib.AcqSpec(kind=kind, obj_scale=1.0)
    buf = C.c_void_p(1 << 20)
    P = {"pending analytic": 1, "33 pending": 33, "null pending": 2}.get(case, 0)
    S = 0 if case == "S 0" else 64
    z = None if case == "null samples" else buf
    pend = None if case == "null pending" else buf
    out = None if case == "null output" else buf
    rc = lib.bb_acq_grad(None if case == "null model" else C.byref(m), C.byref(a), buf, 10, P, pend, pend, pend, pend,
                         z, S, out, out, None)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()
    assert lib.bb_acq_grad(C.byref(_fake()), C.byref(_lib.AcqSpec(kind=0, obj_scale=1.0)), None, 0, 0, None, None,
                           None, None, buf, 64, None, None, None) == 0


# ---- Campaign flows on the stand-in ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bb():
    for p in (str(ROOT / "tests" / "shims"), str(REF)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe_b200 import baybe_plugin, surrogates

    saved = surrogates.DeviceGP
    if not torch.cuda.is_available():
        surrogates.DeviceGP = OracleGradGP
    yield baybe_plugin
    surrogates.DeviceGP = saved


def _space(kind: str, fixed: bool = False):
    from baybe.parameters import CategoricalParameter, NumericalContinuousParameter, NumericalDiscreteParameter
    from baybe.parameters.numerical import _FixedNumericalContinuousParameter
    from baybe.searchspace import SearchSpace

    cont = [NumericalContinuousParameter("temperature", (40.0, 120.0)),
            NumericalContinuousParameter("pressure", (1.0, 5.0))]
    if fixed:
        cont.append(_FixedNumericalContinuousParameter(name="flow", value=2.0))
    if kind == "continuous":
        return SearchSpace.from_product(cont)
    disc = [NumericalDiscreteParameter("time", values=[1, 2, 4]),
            CategoricalParameter("solvent", values=["A", "B"], encoding="OHE")]
    return SearchSpace.from_product(disc + cont)


def _measure(df: pd.DataFrame, rng) -> pd.DataFrame:
    out = df.copy()
    y = -0.002 * (out["temperature"] - 85) ** 2 + 0.8 * out["pressure"] + rng.normal(0, 0.05, len(out))
    if "time" in out:
        y = y + 0.3 * out["time"] + (out["solvent"] == "B") * 0.5
    out["yield"] = y
    return out


def _campaign(plugin, space, acqf=None, **kw):
    from baybe import Campaign
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    d = len(space.comp_rep_columns)
    hyper = {"lengthscale": np.full(d, 0.5), "noise": 1e-3, "mean_const": 0.0}
    extra = {} if acqf is None else {"acquisition_function": acqf}
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hyper),
                                        n_mc_samples=64, n_raw_samples=32, n_restarts=4, **extra, **kw)
    return Campaign(space, SingleTargetObjective(NumericalTarget("yield")), rec)


def _initial(space, n, rng):
    df = space.sample_uniform(n) if hasattr(space, "sample_uniform") else None
    if df is None:
        cont = space.continuous.sample_uniform(n)
        if space.discrete.exp_rep.shape[1]:
            disc = space.discrete.exp_rep.sample(n, replace=True, random_state=int(rng.integers(1 << 30)))
            df = pd.concat([disc.reset_index(drop=True), cont.reset_index(drop=True)], axis=1)
        else:
            df = cont
    return df.reset_index(drop=True)


@needs_ref
@pytest.mark.parametrize("kind", ["continuous", "hybrid"])
def test_campaign_flow_with_the_default_acquisition_function(bb, kind):
    rng = np.random.default_rng(0)
    space = _space(kind, fixed=True)
    camp = _campaign(bb, space)
    camp.add_measurements(_measure(_initial(space, 6, rng), rng))
    rec = camp.recommend(3)
    # the reference's layout: discrete experimental columns first, then the continuous parameters
    assert list(rec.columns) == list(space.discrete.exp_rep.columns) + list(space.continuous.parameter_names)
    assert len(rec) == 3
    assert (rec["flow"] == 2.0).all()
    assert rec["temperature"].between(40, 120).all() and rec["pressure"].between(1, 5).all()
    camp.add_measurements(_measure(rec, rng))
    pend = rec.iloc[:1]
    rec2 = camp.recommend(2, pending_experiments=pend)
    assert len(rec2) == 2
    if kind == "hybrid":
        # the discrete part keeps the search space's index labels; a label may repeat within a batch
        assert set(rec2.index) <= set(space.discrete.exp_rep.index)
        assert rec2["time"].isin([1, 2, 4]).all() and rec2["solvent"].isin(["A", "B"]).all()
    # the acquisition callable values continuous candidates through the existing scoring path
    vals = camp.acquisition_values(rec2)
    assert len(vals) == 2 and np.all(np.isfinite(vals.to_numpy(dtype=float)))
    assert np.isfinite(camp.joint_acquisition_value(rec2))


@needs_ref
def test_rejections(bb):
    from baybe.acquisition import UCB, qNEI
    from baybe.constraints import ContinuousLinearConstraint
    from baybe.exceptions import IncompatibilityError, IncompatibleAcquisitionFunctionError
    from baybe.searchspace import SearchSpace, SubspaceContinuous

    rng = np.random.default_rng(1)
    space = _space("continuous")
    init = _measure(_initial(space, 5, rng), rng)
    camp = _campaign(bb, space, sequential_continuous=False)
    camp.add_measurements(init)
    with pytest.raises(NotImplementedError, match="sequential"):
        camp.recommend(2)
    camp = _campaign(bb, space, acqf=UCB())
    camp.add_measurements(init)
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="batch sizes > 1"):
        camp.recommend(2)
    camp = _campaign(bb, space, acqf=qNEI())
    camp.add_measurements(init)
    with pytest.raises(IncompatibleAcquisitionFunctionError):
        camp.recommend(1)
    cons = ContinuousLinearConstraint(parameters=["temperature", "pressure"], operator="<=", coefficients=[1.0, 1.0],
                                      rhs=100.0)
    cspace = SearchSpace(continuous=SubspaceContinuous(space.continuous.parameters, constraints_lin_ineq=[cons]))
    camp = _campaign(bb, cspace)
    camp.add_measurements(init)
    with pytest.raises(IncompatibilityError, match="constraints"):
        camp.recommend(1)
    with pytest.raises(ValueError, match="between 0 and 1"):
        bb.B200BotorchRecommender(sampling_percentage=1.5)
