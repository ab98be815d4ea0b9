"""CPU tests of the hypervolume acquisition functions (qEHVI / qLogEHVI): the host partitioning against brute-force
hypervolumes, the reference point, the incremental pending form against literal inclusion-exclusion, the argument
checks of ``bb_hvi_score`` and the Campaign glue on a float64 stand-in engine."""
from __future__ import annotations

import ctypes as C
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import multiobjective as mo
from tests import mo_oracle

ROOT = Path(__file__).resolve().parents[1]


# ---- partitioning ---------------------------------------------------------------------------------------------
def _random_front(rng, M, k):
    Y = rng.normal(size=(k, M))
    Y[: k // 4] = np.round(Y[: k // 4], 1)  # ties
    Y = np.concatenate([Y, Y[:2], rng.normal(size=(2, M)) - 3.0])  # duplicates, points below the reference point
    return Y, np.full(M, -1.5)


@pytest.mark.parametrize("M,k,seed", [(2, 9, 0), (2, 1, 1), (3, 8, 2), (3, 12, 3), (4, 6, 4), (4, 9, 5)])
def test_box_decomposition_is_exact(M, k, seed):
    rng = np.random.default_rng(seed)
    Y, ref = _random_front(rng, M, k)
    lo, up, hv = mo.box_decomposition(Y, ref)
    assert abs(hv - mo_oracle.hv(Y, ref)) < 1e-12
    top = np.full(M, 4.0)
    assert (up > lo).all() and (lo >= ref).all()
    lc, uc = np.minimum(lo, top), np.minimum(up, top)
    # pairwise disjoint
    inter = np.clip(np.minimum(uc[:, None], uc[None]) - np.maximum(lc[:, None], lc[None]), 0, None).prod(-1)
    np.fill_diagonal(inter, 0.0)
    assert inter.max() == 0.0
    # volume inside the bounding box = box volume - hv(F)
    assert abs(np.prod(uc - lc, axis=1).sum() - (np.prod(top - ref) - hv)) < 1e-10
    # hard HVI of random points = hv(F u {y}) - hv(F)
    for y in rng.normal(size=(20, M)) * 1.5:
        got = float(mo.hvi_hard(lo, up, y[None])[0])
        assert abs(got - (mo_oracle.hv(np.vstack([Y, y]), ref) - hv)) < 1e-12


def test_empty_front_is_one_open_cell():
    lo, up, hv = mo.box_decomposition(np.zeros((0, 3)), np.zeros(3))
    assert hv == 0.0 and len(lo) == 1 and np.isinf(up).all()


# ---- reference point --------------------------------------------------------------------------------------------
def test_compute_ref_point_matches_the_reference_docstring():
    assert np.allclose(mo.compute_ref_point([[0, 10], [2, 20]], [True, True], 0.1), [-0.2, 9.0])
    assert np.allclose(mo.compute_ref_point([[0, 10], [2, 20]], [True, False], 0.2), [-0.4, 22.0])
    with pytest.raises(ValueError):
        mo.compute_ref_point([1.0, 2.0])


def test_compute_ref_point_equals_baybe():
    ref_dir = ROOT / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    from baybe.acquisition import qLogNEHVI

    rng = np.random.default_rng(0)
    for _ in range(5):
        arr = rng.normal(size=(7, 3))
        mx = rng.random(3) < 0.5
        f = float(rng.uniform(-0.5, 0.5))
        assert np.allclose(mo.compute_ref_point(arr, mx, f), qLogNEHVI.compute_ref_point(arr, mx, f), atol=1e-14)


# ---- pending points and smoothing --------------------------------------------------------------------------------
def _models(M=2, n=10, d=3, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.random((n, d))
    oms = []
    for m in range(M):
        y = np.sin(3 * X @ rng.normal(size=d)) + 0.05 * rng.normal(size=n)
        spec = oracle.KernelSpec(family="matern52", lengthscale=np.full(d, 0.5), active_dims=list(range(d)))
        oms.append(oracle.build_model(spec, X, y, np.stack([np.zeros(d), np.ones(d)]), noise=1e-3, mean_const=0.0))
    a, b = np.array([1.0, -1.0, 1.0][:M]), np.zeros(M)
    front = np.stack([oracle.posterior(om, X)[0].numpy() for om in oms], 1) * a + b
    ref = mo.compute_ref_point(front)
    return oms, a, b, ref, front, rng


@pytest.mark.parametrize("M,P", [(2, 0), (2, 1), (2, 3), (3, 2)])
def test_incremental_qehvi_equals_inclusion_exclusion(M, P):
    oms, a, b, ref, front, rng = _models(M=M, seed=M + P)
    x = rng.random((1, 3))
    pend = rng.random((P, 3)) if P else None
    z = oracle.sobol_normal_samples(64, M * (P + 1), seed=5)
    inc = float(mo_oracle.ehvi(oms, "qEHVI", a, b, ref, front, x, pend, z)[0])
    lit = mo_oracle.inclusion_exclusion(oms, "qEHVI", a, b, ref, front, x, pend, z)
    assert lit > 0 and abs(inc - lit) < 1e-10


# stated bound on |incremental qLogEHVI - literal smoothed inclusion-exclusion| (natural-log units); with P = 0 the
# two forms are the same expression
QLOG_PENDING_TOL = 0.05


@pytest.mark.parametrize("M,P", [(2, 0), (2, 1), (2, 3), (3, 2)])
def test_incremental_qlogehvi_against_smoothed_inclusion_exclusion(M, P):
    oms, a, b, ref, front, rng = _models(M=M, seed=10 + M + P)
    x = rng.random((1, 3))
    pend = rng.random((P, 3)) if P else None
    z = oracle.sobol_normal_samples(64, M * (P + 1), seed=6)
    inc = float(mo_oracle.ehvi(oms, "qLogEHVI", a, b, ref, front, x, pend, z)[0])
    lit = mo_oracle.inclusion_exclusion(oms, "qLogEHVI", a, b, ref, front, x, pend, z)
    print(f"M={M} P={P}: incremental {inc:.6f} literal {lit:.6f} diff {inc - lit:+.2e}")
    assert abs(inc - lit) < (1e-9 if P == 0 else QLOG_PENDING_TOL)


def test_qlogehvi_converges_to_qehvi_as_the_temperatures_shrink():
    oms, a, b, ref, front, rng = _models(M=2, seed=3)
    lo, up, _ = mo.box_decomposition(front, ref)
    Y = torch.as_tensor(rng.normal(size=(200, 2)) + front.mean(0))
    hard = mo_oracle.cell_values(Y, lo, up, log=False)
    errs = []
    for tau in (1e-2, 1e-3, 1e-4):
        soft = mo_oracle.cell_values(Y, lo, up, log=True, tau_relu=tau * 1e-4, tau_max=tau).exp()
        errs.append(float((soft - hard).abs().max()))
    assert errs[2] < errs[1] < errs[0] and errs[2] < 1e-3


# ---- bb_hvi_score argument checks ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _call(lib, **over):
    from baybe_b200 import _lib

    a = _lib.AcqSpec(kind=over.pop("kind", _lib.ACQ_KIND["qLogEHVI"]), tau_relu=over.pop("tau_relu", 1e-6),
                     tau_max=1e-2)
    M = over.pop("M", 2)
    fa = (C.c_float * 4)(1, 1, 1, 1)
    p = C.c_void_p(1 << 20)
    args = dict(a=None if over.pop("null_acq", False) else C.byref(a), M=M, sa=fa, sb=fa, N=100, mu=p, var=p, P=0,
                cross=None, linv=None, w=None, z=p, S=64, lower=p, upper=p, counts=p, stride=8, keep=None, score=p,
                key=p, offset=0, stream=None)
    args.update(over)
    return lib.bb_hvi_score(*args.values())


_BAD = [
    ("null spec", dict(null_acq=True), "invalid", b"spec is null"),
    ("kind qLogEI", dict(kind=0), "invalid", b"not a hypervolume"),
    ("tau_relu 0", dict(tau_relu=0.0), "invalid", b"tau_relu"),
    ("M = 1", dict(M=1), "unsupported", b"n_targets=1"),
    ("M = 5", dict(M=5), "unsupported", b"n_targets=5"),
    ("S = 0", dict(S=0), "invalid", b"S=0"),
    ("S = 1025", dict(S=1025), "invalid", b"S=1025"),
    ("P = 32", dict(P=32), "invalid", b"n_pending=32"),
    ("stride 0", dict(stride=0), "unsupported", b"cell_stride=0"),
    ("stride 1025", dict(stride=1025), "unsupported", b"cell_stride=1025"),
    ("null key", dict(key=None), "invalid", b"null best key"),
    ("null mu", dict(mu=None), "invalid", b"null buffer"),
    ("null cells", dict(counts=None), "invalid", b"null buffer"),
    ("pending without cross", dict(P=2), "invalid", b"need cross"),
    ("negative offset", dict(offset=-1), "invalid", b"32-bit key"),
]


@pytest.mark.parametrize("case,over,status,msg", _BAD, ids=[c for c, *_ in _BAD])
def test_bb_hvi_score_rejects_bad_arguments_before_any_cuda_call(lib, case, over, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    rc = _call(lib, **over)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


def test_bb_hvi_score_accepts_an_empty_candidate_set(lib):
    assert _call(lib, N=0, mu=None, var=None) == 0


def test_too_many_cells_is_a_clear_error():
    lo = np.zeros((1500, 2))
    with pytest.raises(NotImplementedError, match="1500 cells"):
        mo._padded([(lo, lo + 1)], 2)


# ---- Campaign glue on a float64 stand-in engine ------------------------------------------------------------------------
def _hvi_score_f64(mu, var, cross, linv, w, z, lower, upper, n_cells, keep, kind, params, a, b, index_offset,
                   want_scores):
    """Float64 stand-in of ``baybe_b200::hvi_score`` (same arguments, same definition as csrc/mo.cu)."""
    from baybe_b200 import _lib
    from baybe_b200.engine import pack_best

    M, N = mu.shape
    P = 0 if cross is None else cross.shape[2]
    Q = P + 1
    z = z.double()
    S = z.shape[0]
    mu, var = mu.double(), var.double()
    a = torch.tensor(a, dtype=torch.float64)
    b = torch.tensor(b, dtype=torch.float64)
    Y = torch.empty(S, N, M, dtype=torch.float64)
    for m in range(M):
        zx = z[:, m * Q + P]
        if P == 0:
            Y[:, :, m] = mu[m][None] + var[m].clamp_min(0).sqrt()[None] * zx[:, None]
        else:
            c = cross[m].double()
            r2 = (c @ linv[m].double().T).pow(2).sum(1)
            sd = (var[m] - r2).clamp_min(0).sqrt()
            Y[:, :, m] = mu[m][None] + w[m].double() @ c.T + sd[None] * zx[:, None]
    Y = a * Y + b
    log = kind == _lib.ACQ_KIND["qLogEHVI"]
    rows = []
    for s in range(S):
        k = 0 if lower.shape[0] == 1 else s
        nc = int(n_cells[k])
        rows.append(mo_oracle.cell_values(Y[s], lower[k, :nc].double(), upper[k, :nc].double(), log=log))
    v = torch.stack(rows)
    val = (torch.logsumexp(v, 0) - math.log(S)) if log else v.mean(0)
    s32 = val.float()
    best = -(1 << 63)
    for i in range(N):
        if (keep is None or int(keep[i]) != 0) and not math.isnan(float(s32[i])):
            best = max(best, pack_best(float(s32[i]), i + int(index_offset)))
    return (s32 if want_scores else None), torch.tensor([best], dtype=torch.int64)


@pytest.fixture()
def bb(monkeypatch):
    ref_dir = ROOT / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(ROOT / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe_b200 import baybe_plugin, surrogates
    from tests.helpers import OracleBackedGP

    class StandInGP(OracleBackedGP):
        """OracleBackedGP plus the pending-point calls the hypervolume scorer makes."""

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
    monkeypatch.setattr(mo, "_hvi_score", _hvi_score_f64)
    return baybe_plugin


def pareto_campaign(plugin, acqf, targets=None, hp=True):
    """Shared by the CPU and GPU Campaign tests: a 216-row discrete space, yield maximised and cost minimised."""
    from baybe import Campaign
    from baybe.objectives import ParetoObjective
    from baybe.parameters import CategoricalParameter, NumericalDiscreteParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    params = [NumericalDiscreteParameter("temperature", values=[60, 70, 80, 90, 100, 110]),
              NumericalDiscreteParameter("concentration", values=[0.1, 0.2, 0.4, 0.8]),
              CategoricalParameter("solvent", values=["A", "B", "C"], encoding="OHE"),
              NumericalDiscreteParameter("time", values=[1, 2, 4])]
    space = SearchSpace.from_product(params)
    d = len(space.comp_rep_columns)
    hyper = {"lengthscale": np.full(d, 0.9), "noise": 5e-3, "mean_const": 0.0} if hp else None
    targets = targets or [NumericalTarget("yield"), NumericalTarget("cost", minimize=True)]
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hyper),
                                        acquisition_function=acqf, n_mc_samples=128)
    camp = Campaign(space, ParetoObjective(targets), rec, allow_recommending_already_measured=False)
    return camp, space


def measure(df, rng, names=("yield", "cost")):
    out = df.copy()
    s = {"A": 0.0, "B": 1.5, "C": -1.0}
    t = out["temperature"]
    cols = {
        "yield": 50 + 0.2 * (t - 85) - 0.01 * (t - 85) ** 2 + 8 * out["concentration"]
        + out["solvent"].map(s).astype(float),
        "cost": 3.0 + 0.02 * t + 2.0 * out["concentration"] ** 2 + 0.3 * out["time"],
        "purity": 90 - 0.05 * (t - 80) ** 2 / 10 + out["time"],
        "speed": 1.0 / out["time"] + 0.01 * t,
        "waste": out["concentration"] * 3 + 0.1 * out["time"],
    }
    for n in names:
        out[n] = cols[n] + rng.normal(0, 0.05, len(out))
    return out


@pytest.mark.parametrize("kind", ["qLogEHVI", "qEHVI"])
def test_pareto_campaign_on_the_stand_in_engine(bb, kind):
    from baybe.acquisition import acqfs

    rng = np.random.default_rng(0)
    acqf = {"qEHVI": acqfs.qExpectedHypervolumeImprovement, "qLogEHVI": acqfs.qLogExpectedHypervolumeImprovement}[kind]
    camp, space = pareto_campaign(bb, acqf())
    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, rng))
    rec = camp.recommend(batch_size=2)
    assert len(rec) == 2 and rec.index.is_unique and not set(rec.index) & set(seed_rows.index)
    camp.add_measurements(measure(rec, rng))
    torch.manual_seed(11)
    r1 = camp.recommend(batch_size=1)
    torch.manual_seed(11)
    vals = camp.acquisition_values(space.discrete.exp_rep)
    assert vals.index.equals(space.discrete.exp_rep.index)
    remaining = vals.drop(index=list(seed_rows.index) + list(rec.index))
    assert r1.index[0] == remaining.idxmax()
    torch.manual_seed(11)
    jv = camp.joint_acquisition_value(r1)
    assert abs(jv - float(vals.loc[r1.index[0]])) < 1e-4 * max(1.0, abs(jv))
    # pending experiments are conditioned on
    rec3 = camp.recommend(batch_size=2, pending_experiments=r1)
    assert r1.index[0] not in rec3.index


def test_pareto_campaign_rejections(bb):
    from baybe.acquisition import qLogNEHVI
    from baybe.acquisition.acqfs import qExpectedHypervolumeImprovement as qEHVI
    from baybe.acquisition.acqfs import qLogExpectedHypervolumeImprovement as qLogEHVI
    from baybe.exceptions import IncompatibleAcquisitionFunctionError, IncompleteMeasurementsError
    from baybe.targets import NumericalTarget

    rng = np.random.default_rng(2)
    camp, space = pareto_campaign(bb, qLogEHVI())
    rows = measure(space.discrete.exp_rep.sample(10, random_state=3), rng)
    rows.loc[rows.index, "cost"] = [np.nan if i % 2 else v for i, v in enumerate(rows["cost"])]
    rows.loc[rows.index[0::2], "yield"] = np.nan
    camp.add_measurements(rows)
    with pytest.raises(IncompleteMeasurementsError):
        camp.recommend(batch_size=1)
    for acqf in (qEHVI(alpha=0.1), qLogNEHVI()):
        camp, space = pareto_campaign(bb, acqf)
        camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng))
        with pytest.raises(IncompatibleAcquisitionFunctionError, match="qEHVI|alpha"):
            camp.recommend(batch_size=1)
    names = ("yield", "cost", "purity", "speed", "waste")
    camp, space = pareto_campaign(bb, qLogEHVI(), targets=[NumericalTarget(n) for n in names])
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng, names))
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="2 to 4 targets"):
        camp.recommend(batch_size=1)
    # a non-affine target transformation, through the Campaign
    from baybe.transformations import ExponentialTransformation

    camp, space = pareto_campaign(bb, qLogEHVI(), targets=[
        NumericalTarget("yield"), NumericalTarget("cost", transformation=ExponentialTransformation(), minimize=True)])
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng))
    with pytest.raises(NotImplementedError, match="not affine"):
        camp.recommend(batch_size=1)
    # a hypervolume acquisition function on a single-target objective
    from baybe import Campaign
    from baybe.objectives import SingleTargetObjective

    from baybe_b200.surrogates import GaussianProcessSurrogate

    hp = {"lengthscale": np.full(len(space.comp_rep_columns), 0.9), "noise": 5e-3, "mean_const": 0.0}
    single = Campaign(space, SingleTargetObjective(NumericalTarget("yield")), bb.B200BotorchRecommender(
        surrogate_model=GaussianProcessSurrogate(hyperparameters=hp)))
    single.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng, ("yield",)))
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="multi-output"):
        single.acquisition_values(space.discrete.exp_rep.head(5), acquisition_function=qLogEHVI())


def test_acquisition_callable_rejects_more_than_31_other_points_before_scoring(bb, monkeypatch):
    """The joint value of a q-batch with its pending points: up to 31 points besides the candidate are scored, more
    raise NotImplementedError before the scoring op is called."""
    from baybe_b200 import surrogates
    from baybe_b200.engine import AcqConfig

    rng = np.random.default_rng(7)
    X = rng.random((10, 3))
    gps = [surrogates.DeviceGP(X, np.sin(3 * X @ rng.normal(size=3)), np.stack([np.zeros(3), np.ones(3)]),
                               "matern52", 0.5, 1e-3) for _ in range(2)]
    front = np.stack([gp.posterior(X)[0].double().numpy() for gp in gps], 1)
    scorer = mo.HviScorer(gps, AcqConfig(kind="qEHVI"), [1.0, 1.0], [0.0, 0.0], mo.compute_ref_point(front), front)
    calls = []
    monkeypatch.setattr(mo, "_hvi_score", lambda *a: calls.append(1) or _hvi_score_f64(*a))
    pend = torch.from_numpy(rng.random((29, 3)))
    acqf = bb.EngineAcquisitionFunction(None, scorer.cfg, 8, X_pending=pend, scorer=scorer)
    with pytest.raises(NotImplementedError, match="at most 32 points"):
        acqf(torch.from_numpy(rng.random((1, 4, 3))))  # 3 batch + 29 pending points besides the candidate
    assert not calls
    assert np.isfinite(float(acqf(torch.from_numpy(rng.random((1, 3, 3))))[0])) and len(calls) == 1


def test_grid_work_is_bounded_before_the_grid_is_built():
    F = np.random.default_rng(0).normal(size=(400, 4))
    F = F / np.linalg.norm(F, axis=1, keepdims=True)  # points on a sphere: most are non-dominated
    with pytest.raises(NotImplementedError, match="column-point tests"):
        mo.box_decomposition(np.abs(F), np.zeros(4))


def check_subset_batch_wins(plugin, monkeypatch, rng, acqf):
    """Pareto campaign with a subset-generating constraint (``DiscreteBatchConstraint``): the batch shares one value
    of the constrained parameter and is, of the per-subset batches, the one with the highest joint value.  Shared by
    the stand-in test below and tests/test_gpu_mo.py."""
    from baybe import Campaign
    from baybe.constraints import DiscreteBatchConstraint
    from baybe.objectives import ParetoObjective
    from baybe.parameters import CategoricalParameter, NumericalDiscreteParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate

    params = [NumericalDiscreteParameter("x", values=[0.0, 0.25, 0.5, 0.75, 1.0]),
              NumericalDiscreteParameter("y", values=[0.0, 0.5, 1.0]),
              CategoricalParameter("cat", values=["p", "q", "r"], encoding="OHE")]
    space = SearchSpace.from_product(params, constraints=[DiscreteBatchConstraint(parameters=["cat"])])
    assert space.discrete.n_subsets > 0
    d = len(space.comp_rep_columns)
    hp = {"lengthscale": np.full(d, 0.7), "noise": 1e-2, "mean_const": 0.0}
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp),
                                        acquisition_function=acqf, n_mc_samples=128)
    camp = Campaign(space, ParetoObjective([NumericalTarget("t1"), NumericalTarget("t2", minimize=True)]), rec)
    rows = space.discrete.exp_rep.sample(8, random_state=0)
    meas = rows.copy()
    shift = rows["cat"].map({"p": 0.0, "q": 0.3, "r": -0.2}).astype(float)
    meas["t1"] = rows["x"] - (rows["y"] - 0.5) ** 2 + shift + rng.normal(0, 0.02, len(rows))
    meas["t2"] = rows["x"] ** 2 + rows["y"] - shift + rng.normal(0, 0.02, len(rows))
    camp.add_measurements(meas)
    batches, values = [], []
    without = plugin.B200BotorchRecommender._recommend_discrete_without_subsets
    call = plugin.EngineAcquisitionFunction.__call__

    def spy_batch(self, *args):
        idx = without(self, *args)
        batches.append(list(idx))
        return idx

    def spy_value(self, X):
        out = call(self, X)
        values.append(float(out[0]))
        return out

    monkeypatch.setattr(plugin.B200BotorchRecommender, "_recommend_discrete_without_subsets", spy_batch)
    monkeypatch.setattr(plugin.EngineAcquisitionFunction, "__call__", spy_value)
    batch = camp.recommend(batch_size=3)
    assert len(batch) == 3 and batch["cat"].nunique() == 1
    assert len(batches) == len(values) >= 2
    assert list(batch.index) == batches[int(np.argmax(values))]


def test_pareto_subset_constraint_on_the_stand_in_engine(bb, monkeypatch):
    from baybe.acquisition.acqfs import qLogExpectedHypervolumeImprovement

    check_subset_batch_wins(bb, monkeypatch, np.random.default_rng(5), qLogExpectedHypervolumeImprovement())
