"""CPU tests of qLogNParEGO on discrete spaces: the simplex weights against botorch's recipe, the Chebyshev
scalarisation and its degenerate range, the baseline pruning against a brute-force restatement, the conditional value
against the full joint Cholesky of [C; x] per target, the tau limit, invariances of the recommendation, q-batch joint
values, the argument checks of ``bb_parego_score`` and the Campaign glue on a float64 stand-in engine."""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import noisy, parego
from baybe_b200.engine import AcqConfig, sobol_normal_samples
from baybe_b200.synthetic import numeric_grid_workload
from tests import parego_oracle as po
from tests.test_nei import _brute_prune

ROOT = Path(__file__).resolve().parents[1]
CFG = AcqConfig(kind="qLogNParEGO")


@pytest.fixture()
def f64_engine(monkeypatch):
    monkeypatch.setattr(noisy, "_joint_posterior", po.joint_posterior_f64)
    monkeypatch.setattr(parego, "_parego_score", po.parego_score_f64)


def _scorer(M=2, n=20, seed=0, N=300, d=4, prune=True, prune_seed=1, scales=None, shifts=None, weights=None, **kw):
    w = numeric_grid_workload(N=N, d=d, n=n, seed=seed)
    gps = po.stand_in_models(w, M, seed=seed)
    a = np.array(scales if scales is not None else [1.0, -1.0] * (M // 2) + [1.0] * (M % 2))
    b = np.array(shifts if shifts is not None else np.linspace(0.0, 0.5, M))
    lam = np.asarray(weights) if weights is not None else np.linspace(1.0, 2.0, M) / np.linspace(1.0, 2.0, M).sum()
    cfg = dataclasses.replace(CFG, **kw)
    return w, gps, parego.ParegoScorer(gps, cfg, a, b, w.train_x, lam, prune=prune, prune_seed=prune_seed)


def _unmeasured(w, k, seed):
    X = w.candidates  # a measured candidate would make the joint covariance of [C; x] singular
    X = X[np.abs(X[:, None, :] - w.train_x[None]).sum(-1).min(1) > 1e-9]
    return X[np.random.default_rng(seed).choice(len(X), k, replace=False)]


# ---- weights and scalarisation ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [2, 5, 8])
def test_weights_follow_botorchs_simplex_recipe(M):
    torch.manual_seed(5)
    lam = parego.sample_simplex(M)
    torch.manual_seed(5)
    u = torch.rand(1, M - 1, dtype=torch.float64)[0].numpy()
    edges = np.concatenate([[0.0], np.sort(u), [1.0]])
    assert np.array_equal(lam, edges[1:] - edges[:-1])
    assert lam.shape == (M,) and (lam >= 0).all() and abs(lam.sum() - 1.0) < 1e-15
    assert not np.array_equal(lam, parego.sample_simplex(M))  # a fresh draw per construction


def test_chebyshev_is_the_literal_formula():
    p = np.random.default_rng(0).normal(size=(7, 3, 5))
    ref = np.empty((7, 3))
    for i in range(7):
        for j in range(3):
            ref[i, j] = min(p[i, j]) + 0.05 * sum(p[i, j])
    assert np.allclose(parego.chebyshev(p), ref, rtol=0, atol=1e-15)


def test_normalisation_and_the_degenerate_range(f64_engine):
    w, gps, sc = _scorer(M=3, scales=[2.0, -1.0, 1.0], shifts=[0.5, 3.0, -1.0])
    o = np.stack([po.joint_posterior_f64(g, w.train_x)[0] for g in gps], 1) * sc.a + sc.b
    lo, hi = o.min(0), o.max(0)
    p = sc.W * np.stack([po.joint_posterior_f64(g, w.train_x)[0] for g in gps], 1) + sc.V
    assert np.allclose(p, sc.weights * (o - lo) / (hi - lo), atol=1e-13)
    # one measured row: every range is 0 and counts as 1, so p_m = lambda_m (o_m - o_m(x_1))
    one = parego.ParegoScorer(gps, CFG, sc.a, sc.b, w.train_x[:1], sc.weights)
    o1 = np.array([po.joint_posterior_f64(g, w.train_x[:1])[0][0] for g in gps]) * sc.a + sc.b
    assert np.allclose(one.W, sc.weights * sc.a) and np.allclose(one.V, sc.weights * (sc.b - o1))
    assert list(one.winners) == [0] and np.isfinite(one.scores(w.candidates[:5], None, seed=0, n_samples=32)).all()


# ---- pruning -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [2, 5])
def test_pruning_keeps_the_winners_of_the_scalarised_joint_samples(f64_engine, M):
    w, gps, sc = _scorer(M=M, n=30, prune_seed=3)
    n = 30
    z = sobol_normal_samples(noisy.PRUNE_SAMPLES, M * n, 3).numpy()
    Y = np.empty((noisy.PRUNE_SAMPLES, n, M))
    for m, g in enumerate(gps):  # column m n + i of the Sobol draw is row i of target m
        mu, cov = oracle.posterior_joint(g.om, w.train_x)
        Y[:, :, m] = mu.numpy()[None] + z[:, m * n:(m + 1) * n] @ np.linalg.cholesky(cov.numpy()).T
    P = sc.W * Y + sc.V
    cheb = np.array([[min(r) + 0.05 * sum(r) for r in s] for s in P])
    assert list(sc.winners) == sorted(set(int(np.argmax(r)) for r in cheb))
    assert 1 < len(sc.winners) < n
    for n_other in (0, 25, 29):
        cap = 31 - n_other
        kept = sc.kept_baseline(n_other)
        assert list(kept) == _brute_prune(cheb, cap)
        assert sc.n_dropped == len(sc.winners) - len(kept)


def test_prune_baseline_false_conditions_on_every_row_up_to_the_limit(f64_engine):
    w, gps, sc = _scorer(M=3, n=29, prune=False)
    assert list(sc.kept_baseline(2)) == list(range(29)) and sc.n_dropped == 0
    with pytest.raises(NotImplementedError, match="prune_baseline=False.*at most 31"):
        sc.kept_baseline(3)
    with pytest.raises(NotImplementedError, match="at most 31"):
        sc.joint_value(w.candidates[:4], None, seed=0, n_samples=16)


# ---- the value ----------------------------------------------------------------------------------------------------------------
def _setup(M, P, Q, n=20, seed=0, **kw):
    w, gps, sc = _scorer(M=M, n=n, seed=seed, **kw)
    X = _unmeasured(w, P + Q + 30, seed + 10)
    return w, gps, sc, (X[:P] if P else None), (X[P:P + Q] if Q else None), X[P + Q:]


def _conditional(sc, gps, pend, batch, x, S=64, seed=7, log=True):
    n_other = (0 if pend is None else len(pend)) + (0 if batch is None else len(batch))
    nc = sc.n_conditioning(n_other)
    M = sc.M
    z = sobol_normal_samples(S, M * (1 + nc), seed).numpy()
    rows, linv, w, g, terms, _ = sc.conditioning(pend, batch, z)
    mu, var, cross = [], [], []
    for gp in gps:
        m_, v_ = oracle.posterior(gp.om, x)
        _, cov = oracle.posterior_joint(gp.om, np.concatenate([rows, x]))
        mu.append(m_), var.append(v_), cross.append(cov[nc:, :nc])
    zx = np.stack([z[:, m * (nc + 1) + nc] for m in range(M)], 1)
    c = sc.cfg
    val = po.parego_values_f64(torch.stack(mu), torch.stack(var), torch.stack(cross), linv, w.transpose(0, 2, 1), zx,
                               g, terms, sc.W, sc.V, sc.alpha, c.tau_relu, c.tau_max, log=log)
    return val, rows, z, nc


@pytest.mark.parametrize("M", [2, 5])
@pytest.mark.parametrize("P,Q", [(0, 0), (3, 0), (0, 2), (4, 3)])
def test_conditional_value_equals_the_full_joint_cholesky(f64_engine, M, P, Q):
    w, gps, sc, pend, batch, x = _setup(M, P, Q)
    val, rows, z, nc = _conditional(sc, gps, pend, batch, x)
    ref = po.parego_full_joint([g.om for g in gps], rows, nc - Q, x, z, sc.W, sc.V, sc.alpha, sc.cfg.tau_relu,
                               sc.cfg.tau_max)
    assert torch.allclose(val, ref, rtol=1e-10, atol=1e-10), float((val - ref).abs().max())


def test_exp_qlognparego_tends_to_the_hard_value_as_tau_shrinks(f64_engine):
    errs = []
    for tau in (1e-2, 1e-4, 1e-6):
        _, gps, sc, pend, _, x = _setup(3, 2, 0, tau_relu=tau, tau_max=tau)
        lv = torch.from_numpy(sc.scores(x, pend, seed=7, n_samples=64))
        hard, *_ = _conditional(sc, gps, pend, None, x, log=False)
        ok = hard > 1e-3 * float(hard.max())  # relative error where the hard value is not vanishingly small
        assert int(ok.sum()) >= 10
        errs.append(float(((lv.exp() - hard).abs()[ok] / hard[ok]).max()))
    assert errs[0] > errs[1] > errs[2] and errs[2] < 1e-3, errs


def _rebuilt(w, gps, sc, m, y_map, scale_m=None):
    """The same scorer with target m's measurements replaced by y_map(y) (and its orientation scale by scale_m)."""
    new = list(gps)
    new[m] = po.StandInGP(**dataclasses.replace(w, train_y=y_map(gps[m].train_y), noise=np.array([1e-2])).gp_kwargs())
    a = sc.a.copy()
    if scale_m is not None:
        a[m] = scale_m
    return parego.ParegoScorer(new, sc.cfg, a, sc.b, w.train_x, sc.weights)


def test_recommendation_is_invariant_to_affine_rescaling_and_to_flipping_a_target(f64_engine):
    """Standardize makes the posterior of 3y + 5 the affine image of y's and the baseline normalisation removes the
    scale and shift, sample by sample.  Negating the measurements of a target flipped to minimize=True leaves its
    orientation o = y in distribution (the same base samples then draw the mirrored paths), so the recommendation
    stays.  tau_relu = 1e-3: the fp32 moments handed to the kernel round differently for the rescaled target, which
    at tau_relu = 1e-6 moves the values of rows whose improvement sits in the far tail."""
    w, gps, sc = _scorer(M=3, n=20, scales=[1.0, 1.0, 1.0], shifts=[0.0, 0.0, 0.0], tau_relu=1e-3)
    x = _unmeasured(w, 200, 4)
    pend = x[:2]
    ref = sc.scores(x, None, seed=3, n_samples=512)
    ref_p = sc.scores(x, pend, seed=3, n_samples=512)
    scaled = _rebuilt(w, gps, sc, 1, lambda y: 3.0 * y + 5.0)
    flipped = _rebuilt(w, gps, sc, 2, lambda y: -y, -1.0)
    assert np.allclose(scaled.scores(x, None, seed=3, n_samples=512), ref, rtol=1e-4, atol=1e-4)
    for alt in (scaled, flipped):
        assert list(alt.winners) == list(sc.winners)
        assert int(np.argmax(alt.scores(x, None, seed=3, n_samples=512))) == int(np.argmax(ref))
        assert int(np.argmax(alt.scores(x, pend, seed=3, n_samples=512))) == int(np.argmax(ref_p))


def test_joint_value_of_a_q_batch_matches_brute_force(f64_engine):
    w, gps, sc, pend, _, x = _setup(3, 2, 0)
    for q in (1, 2, 4):
        batch = x[:q]
        v = sc.joint_value(batch, pend, seed=4, n_samples=64)
        nc = sc.n_conditioning(2 + q - 1)
        z = sobol_normal_samples(64, 3 * (1 + nc), 4).numpy()
        kept = sc.baseline[sc.kept_baseline(2 + q - 1)]
        rows = np.concatenate([kept, pend, batch[1:]])
        ref = float(po.parego_full_joint([g.om for g in gps], rows, len(kept) + 2, batch[:1], z, sc.W, sc.V,
                                         sc.alpha, sc.cfg.tau_relu, sc.cfg.tau_max)[0])
        assert abs(v - ref) <= 1e-6 * max(1.0, abs(ref)), (q, v, ref)
    assert sc.joint_value(x[:1], pend, seed=4, n_samples=64) == sc.scores(x[:1], pend, seed=4, n_samples=64)[0]


def test_greedy_rounds_add_the_winner_to_the_conditioning_set(f64_engine):
    from baybe_b200.recommenders import greedy_select

    w, gps, sc, _, _, x = _setup(2, 0, 0)
    chosen, vals = greedy_select(sc, sc.cfg, torch.from_numpy(x), x.shape[1], 3, None, seed=2, n_samples=64)
    assert len(set(chosen)) == 3
    for r in range(3):
        ref = sc.scores(x, x[chosen[:r]] if r else None, seed=2, n_samples=64)
        assert abs(ref[chosen[r]] - vals[r]) <= 1e-6 * max(1.0, abs(vals[r]))
        ref[chosen[:r]] = -np.inf
        assert int(np.argmax(ref)) == chosen[r]


def test_scorer_rejects_target_counts_outside_2_to_8(f64_engine):
    from baybe_b200.acquisition import IncompatibleAcquisitionFunctionError

    w = numeric_grid_workload(N=50, d=3, n=6, seed=0)
    for M in (1, 9):
        gps = po.stand_in_models(w, M)
        with pytest.raises((IncompatibleAcquisitionFunctionError, Exception), match="2 to 8 targets"):
            parego.ParegoScorer(gps, CFG, np.ones(M), np.zeros(M), w.train_x, np.full(M, 1.0 / M))


def test_parego_kind_stays_off_the_fused_kernels():
    from baybe_b200.acquisition import convert_acqf, qLogNParEGO

    spec = convert_acqf("qLogNParEGO")
    assert isinstance(spec, qLogNParEGO) and spec.prune_baseline and spec.supports_multi_output
    assert spec.supports_batching and spec.supports_pending_experiments
    assert CFG.is_mc
    with pytest.raises(NotImplementedError):
        CFG.to_c()


# ---- argument checks ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _call(lib, **over):
    p = C.c_void_p(1 << 20)
    args = dict(M=3, W=(C.c_float * 8)(*([0.3] * 8)), V=(C.c_float * 8)(*([0.1] * 8)), alpha=C.c_float(0.05),
                tau_relu=C.c_float(1e-6), tau_max=C.c_float(1e-2), N=100, mu=p, var=p, C=3, cross=p, linv=p, w=p, z=p,
                S=64, g=p, Q=0, terms=None, keep=None, score=p, key=p, offset=0, stream=None)
    args.update(over)
    return lib.bb_parego_score(*args.values())


_nan_w = (C.c_float * 8)(0.3, math.nan, 0.3, 0.3, 0.3, 0.3, 0.3, 0.3)
_inf_v = (C.c_float * 8)(0.1, 0.1, math.inf, 0.1, 0.1, 0.1, 0.1, 0.1)
_BAD = [
    ("one target", dict(M=1), "unsupported", b"n_targets=1"),
    ("nine targets", dict(M=9), "unsupported", b"n_targets=9"),
    ("null weights", dict(W=None), "invalid", b"null scalarisation"),
    ("weight not finite", dict(W=_nan_w), "invalid", b"target 1 not finite"),
    ("offset not finite", dict(V=_inf_v), "invalid", b"target 2 not finite"),
    ("alpha not finite", dict(alpha=C.c_float(math.inf)), "invalid", b"alpha not finite"),
    ("tau_relu 0", dict(tau_relu=C.c_float(0.0)), "invalid", b"tau_relu"),
    ("tau_max negative", dict(tau_max=C.c_float(-1.0)), "invalid", b"tau_max"),
    ("negative offset", dict(offset=-1), "invalid", b"32-bit key"),
    ("index overflow", dict(N=1 << 32), "invalid", b"32-bit key"),
    ("n_cond 32", dict(C=32), "invalid", b"n_cond=32"),
    ("n_cond -1", dict(C=-1), "invalid", b"n_cond=-1"),
    ("batch above n_cond", dict(Q=4), "invalid", b"n_batch=4"),
    ("S = 0", dict(S=0), "invalid", b"S=0"),
    ("S = 1025", dict(S=1025), "invalid", b"S=1025"),
    ("null key", dict(key=None), "invalid", b"null best key"),
    ("null mu", dict(mu=None), "invalid", b"null buffer"),
    ("null incumbents", dict(g=None), "invalid", b"null buffer"),
    ("conditioning without w", dict(w=None), "invalid", b"need cross, linv and w"),
    ("batch without terms", dict(Q=2), "invalid", b"need their terms"),
]


@pytest.mark.parametrize("case,over,status,msg", _BAD, ids=[c for c, *_ in _BAD])
def test_bb_parego_score_rejects_bad_arguments_before_any_cuda_call(lib, case, over, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    assert _call(lib, **over) == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


def test_bb_parego_score_accepts_an_empty_candidate_set(lib):
    assert _call(lib, N=0, mu=None, var=None, g=None) == 0


# ---- Campaign glue on a float64 stand-in engine ----------------------------------------------------------------------------
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

    monkeypatch.setattr(surrogates, "DeviceGP", po.StandInGP)
    return baybe_plugin


NAMES = ("yield", "cost", "purity", "speed", "waste")


def check_parego_flow(plugin, monkeypatch, n_targets, tol):
    """Shared by the CPU and GPU Campaign tests: a Pareto campaign of `n_targets` targets with qLogNParEGO through
    recommend (a greedy batch of 3, then one row, then pending experiments), ``acquisition_values`` (its arg-max is the
    recommended row under the same seeds) and ``joint_acquisition_value``; a fresh campaign with the same data and
    seed recommends the same batch."""
    from baybe.acquisition.acqfs import qLogNParEGO
    from baybe.targets import NumericalTarget

    from baybe_b200 import baybe_plugin, recommenders
    from tests.test_mo import measure, pareto_campaign

    names = NAMES[:n_targets]
    targets = [NumericalTarget(n, minimize=(n in ("cost", "waste"))) for n in names]
    rng = np.random.default_rng(0)
    batches = []
    for _ in range(2):  # the same data and seed in a fresh campaign give the same batch
        camp, space = pareto_campaign(plugin, qLogNParEGO(), targets=targets)
        seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
        camp.add_measurements(measure(seed_rows, np.random.default_rng(0), names))
        torch.manual_seed(3)
        batches.append(camp.recommend(batch_size=3))
    rec = batches[0]
    assert list(batches[1].index) == list(rec.index)
    assert len(rec) == 3 and rec.index.is_unique and not set(rec.index) & set(seed_rows.index)
    scorer = camp.recommender._scorer
    assert isinstance(scorer, parego.ParegoScorer) and scorer.M == n_targets
    assert abs(scorer.weights.sum() - 1.0) < 1e-12 and (scorer.weights >= 0).all()
    camp.add_measurements(measure(rec, rng, names))
    # one sampler seed for every draw, so that recommend and the diagnostics score with the same base samples; the
    # simplex weights come from torch's global RNG, seeded the same way before each call
    for mod in (recommenders, baybe_plugin):
        monkeypatch.setattr(mod, "_draw_sampler_seed", lambda: 77)
    torch.manual_seed(11)
    r1 = camp.recommend(batch_size=1)
    torch.manual_seed(11)
    vals = camp.acquisition_values(space.discrete.exp_rep)
    assert np.isfinite(vals.to_numpy()).all()
    remaining = vals.drop(index=list(seed_rows.index) + list(rec.index))
    assert float(vals.loc[r1.index[0]]) >= float(remaining.max()) - tol * max(1.0, abs(float(remaining.max())))
    torch.manual_seed(11)
    jv = camp.joint_acquisition_value(r1)
    assert abs(jv - float(vals.loc[r1.index[0]])) <= tol * max(1.0, abs(jv))
    torch.manual_seed(12)
    with_pending = camp.acquisition_values(space.discrete.exp_rep.head(20), pending_experiments=r1)
    torch.manual_seed(12)
    assert not np.allclose(with_pending.to_numpy(), camp.acquisition_values(space.discrete.exp_rep.head(20)))
    rec3 = camp.recommend(batch_size=3, pending_experiments=r1)
    assert len(rec3) == 3 and r1.index[0] not in rec3.index
    return camp


@pytest.mark.parametrize("n_targets", [2, 5])
def test_parego_campaign_on_the_stand_in_engine(bb, monkeypatch, n_targets):
    monkeypatch.setattr(parego, "_parego_score", po.parego_score_f64)
    check_parego_flow(bb, monkeypatch, n_targets, tol=0.0)


def test_parego_subset_constraint_on_the_stand_in_engine(bb, monkeypatch):
    from baybe.acquisition.acqfs import qLogNParEGO

    from tests.test_mo import check_subset_batch_wins

    check_subset_batch_wins(bb, monkeypatch, np.random.default_rng(5), qLogNParEGO())


def test_parego_rejections(bb):
    from baybe import Campaign
    from baybe.acquisition.acqfs import qLogNParEGO
    from baybe.exceptions import IncompatibleAcquisitionFunctionError
    from baybe.objectives import ParetoObjective, SingleTargetObjective
    from baybe.parameters import NumericalContinuousParameter, NumericalDiscreteParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget
    from baybe.transformations import ExponentialTransformation

    from baybe_b200.surrogates import GaussianProcessSurrogate
    from tests.test_mo import measure, pareto_campaign

    rng = np.random.default_rng(2)
    # a single-target objective
    camp, space = pareto_campaign(bb, qLogNParEGO())
    hp = {"lengthscale": np.full(len(space.comp_rep_columns), 0.9), "noise": 5e-3, "mean_const": 0.0}
    single = Campaign(space, SingleTargetObjective(NumericalTarget("yield")), bb.B200BotorchRecommender(
        surrogate_model=GaussianProcessSurrogate(hyperparameters=hp)))
    single.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng, ("yield",)))
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="multi-output"):
        single.acquisition_values(space.discrete.exp_rep.head(5), acquisition_function=qLogNParEGO())
    # nine targets
    names = [f"t{i}" for i in range(9)]
    camp, space = pareto_campaign(bb, qLogNParEGO(), targets=[NumericalTarget(n) for n in names])
    rows = space.discrete.exp_rep.sample(10, random_state=3)
    for i, n in enumerate(names):
        rows[n] = rng.normal(size=len(rows)) + i
    camp.add_measurements(rows)
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="2 to 8 targets"):
        camp.recommend(batch_size=1)
    # a target that is not affine
    camp, space = pareto_campaign(bb, qLogNParEGO(), targets=[
        NumericalTarget("yield"), NumericalTarget("cost", transformation=ExponentialTransformation(), minimize=True)])
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng))
    with pytest.raises(NotImplementedError, match="not affine"):
        camp.recommend(batch_size=1)
    # a hybrid space
    space = SearchSpace.from_product([NumericalDiscreteParameter("a", values=[0.0, 0.5, 1.0]),
                                      NumericalContinuousParameter("b", bounds=(0.0, 1.0))])
    hp = {"lengthscale": np.full(2, 0.9), "noise": 5e-3, "mean_const": 0.0}
    camp = Campaign(space, ParetoObjective([NumericalTarget("t1"), NumericalTarget("t2", minimize=True)]),
                    bb.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp),
                                              acquisition_function=qLogNParEGO()))
    meas = space.discrete.exp_rep.sample(3, random_state=0, replace=True).reset_index(drop=True)
    meas["b"], meas["t1"], meas["t2"] = [0.2, 0.5, 0.9], [0.1, 0.4, 0.3], [1.0, 0.2, 0.5]
    camp.add_measurements(meas)
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="discrete search spaces only"):
        camp.recommend(batch_size=1)
