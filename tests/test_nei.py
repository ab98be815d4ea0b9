"""CPU tests of qNEI / qLogNEI on discrete spaces: the baseline pruning rule against a brute-force restatement, the
conditional value against the full joint Cholesky of [C; x], the limits of the conditioning set, the argument checks
of ``bb_nei_score`` and ``bb_joint_posterior``, and the Campaign glue on a float64 stand-in engine."""
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
from baybe_b200 import noisy
from baybe_b200.engine import AcqConfig, sobol_normal_samples
from baybe_b200.synthetic import numeric_grid_workload
from tests import nei_oracle as no

ROOT = Path(__file__).resolve().parents[1]


# ---- pruning ----------------------------------------------------------------------------------------------------------
def _brute_prune(o: np.ndarray, cap: int) -> list[int]:
    counts: dict[int, int] = {}
    for row in o:
        best = 0
        for j in range(1, len(row)):
            if row[j] > row[best]:
                best = j
        counts[best] = counts.get(best, 0) + 1
    order = sorted(counts, key=lambda i: (-counts[i], i))  # most frequent first, ties by index
    return sorted(order[:cap])


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("cap", [1, 3, 8, 31])
def test_pruning_rule_matches_brute_force_with_ties(seed, cap):
    rng = np.random.default_rng(seed)
    o = rng.integers(0, 4, size=(300, 40)).astype(np.float64)  # small integers: ties in most samples
    o[:, 7] += rng.integers(0, 2, size=300)
    winners, counts = noisy.prune_winners(o)
    assert list(winners) == sorted(set(int(np.argmax(r)) for r in o))
    assert list(noisy.kept_points(winners, counts, cap)) == _brute_prune(o, cap)


def _stand_in(n=20, noise=1e-2, seed=0, N=300, d=4):
    w = numeric_grid_workload(N=N, d=d, n=n, seed=seed)
    w = dataclasses.replace(w, noise=np.array([noise]))
    return w, no.StandInGP(**w.gp_kwargs())


@pytest.fixture()
def f64_engine(monkeypatch):
    monkeypatch.setattr(noisy, "_joint_posterior", no.joint_posterior_f64)
    monkeypatch.setattr(noisy, "_nei_score", no.nei_score_f64)


def test_kept_set_is_capped_at_31_minus_the_other_points(f64_engine):
    w, gp = _stand_in(n=40)
    sc = noisy.NeiScorer(gp, AcqConfig(kind="qNEI"), w.train_x)
    sc.winners, sc.counts = np.arange(40), np.arange(40) % 5 + 1  # 40 winners, 8 of them with the top count
    for P in (0, 5, 30):
        kept = sc.kept_baseline(P)
        assert len(kept) == 31 - P and sc.n_dropped == 40 - (31 - P)
        assert list(kept) == noisy.kept_points(sc.winners, sc.counts, 31 - P).tolist()
    with pytest.raises(NotImplementedError, match="at most 31"):
        sc.kept_baseline(31)
    sc.winners, sc.counts = np.array([3, 9]), np.array([5, 7])
    assert list(sc.kept_baseline(4)) == [3, 9] and sc.n_dropped == 0


def test_pruning_keeps_the_sample_winners_of_the_joint_posterior(f64_engine):
    w, gp = _stand_in(n=30, noise=0.2)
    sc = noisy.NeiScorer(gp, AcqConfig(kind="qLogNEI", obj_scale=-1.0), w.train_x, prune_seed=3)
    mu, cov = oracle.posterior_joint(gp.om, w.train_x)
    z = sobol_normal_samples(noisy.PRUNE_SAMPLES, 30, 3).numpy()
    o = -(mu.numpy()[None] + z @ np.linalg.cholesky(cov.numpy()).T)
    assert list(sc.winners) == sorted(set(int(np.argmax(r)) for r in o))
    assert 1 <= len(sc.winners) < 30


def test_prune_baseline_false_conditions_on_every_row_up_to_the_limit(f64_engine):
    w, gp = _stand_in(n=29)
    sc = noisy.NeiScorer(gp, AcqConfig(kind="qNEI"), w.train_x, prune=False)
    assert list(sc.kept_baseline(2)) == list(range(29)) and sc.n_dropped == 0
    with pytest.raises(NotImplementedError, match="prune_baseline=False.*at most 31"):
        sc.kept_baseline(3)


# ---- the value ----------------------------------------------------------------------------------------------------------
def _setup(kind, P, Q, n=20, tau_relu=1e-6, tau_max=1e-2, seed=0):
    w, gp = _stand_in(n=n, seed=seed)
    cfg = AcqConfig(kind=kind, obj_scale=-1.5, obj_shift=0.3, tau_relu=tau_relu, tau_max=tau_max)
    sc = noisy.NeiScorer(gp, cfg, w.train_x, prune_seed=1)
    rng = np.random.default_rng(seed + 10)
    X = w.candidates  # unmeasured rows: a measured candidate would make the joint covariance of [C; x] singular
    X = X[np.abs(X[:, None, :] - w.train_x[None]).sum(-1).min(1) > 1e-9]
    idx = rng.choice(len(X), P + Q + 40, replace=False)
    pend = X[idx[:P]] if P else None
    batch = X[idx[P:P + Q]] if Q else None
    x = X[idx[P + Q:]]
    return w, gp, sc, pend, batch, x


def _conditional(sc, gp, pend, batch, x, S=64, seed=7):
    n_other = (0 if pend is None else len(pend)) + (0 if batch is None else len(batch))
    nc = sc.n_conditioning(n_other)
    z = sobol_normal_samples(S, 1 + nc, seed).numpy()
    rows, linv, w, g, terms, _ = sc.conditioning(pend, batch, z)
    mu, var = oracle.posterior(gp.om, x)
    _, cov = oracle.posterior_joint(gp.om, np.concatenate([rows, x]))
    c = sc.cfg
    val = no.nei_values_f64(mu, var, cov[nc:, :nc], linv, w.T, z[:, nc], g, terms, c.kind == "qLogNEI", c.obj_scale,
                            c.obj_shift, c.tau_relu, c.tau_max)
    return val, rows, z, nc


@pytest.mark.parametrize("kind", ["qNEI", "qLogNEI"])
@pytest.mark.parametrize("P,Q", [(0, 0), (3, 0), (0, 2), (4, 3)])
def test_conditional_value_equals_the_full_joint_cholesky(f64_engine, kind, P, Q):
    w, gp, sc, pend, batch, x = _setup(kind, P, Q)
    val, rows, z, nc = _conditional(sc, gp, pend, batch, x)
    c = sc.cfg
    ref = no.nei_full_joint(gp.om, rows, nc - Q, x, z, kind == "qLogNEI", c.obj_scale, c.obj_shift, c.tau_relu,
                            c.tau_max)
    assert torch.allclose(val, ref, rtol=1e-10, atol=1e-10), float((val - ref).abs().max())


def test_exp_qlognei_converges_to_qnei_as_tau_shrinks(f64_engine):
    errs = []
    for tau in (1e-2, 1e-4, 1e-6):
        _, gp, sc, pend, batch, x = _setup("qLogNEI", 2, 2, tau_relu=tau, tau_max=tau)
        lv = torch.from_numpy(sc.scores(x, pend, seed=7, n_samples=64, batch=batch))
        sc.cfg = dataclasses.replace(sc.cfg, kind="qNEI")
        v = torch.from_numpy(sc.scores(x, pend, seed=7, n_samples=64, batch=batch))
        ok = v > 1e-3 * float(v.max())  # relative error where qNEI is not vanishingly small
        assert int(ok.sum()) >= 10
        errs.append(float(((lv.exp() - v).abs()[ok] / v[ok]).max()))
    assert errs[0] > errs[1] > errs[2] and errs[2] < 1e-3, errs


def test_qnei_with_a_zero_variance_baseline_is_qei_at_the_best_mean(f64_engine, monkeypatch):
    w, gp, sc, _, _, x = _setup("qNEI", 0, 0)

    def noiseless(g, rows, with_beta=False):  # the baseline is known exactly: no variance, no covariance with x
        mu, _, cond = no.joint_posterior_f64(g, rows, with_beta)
        return mu, 1e-30 * np.eye(len(rows)), cond

    def uncorrelated(x_, pend_x, beta):
        mu_, var_ = oracle.posterior(gp.om, np.asarray(x_, dtype=np.float64))
        return mu_.float(), var_.float(), torch.zeros(len(mu_), len(pend_x))

    monkeypatch.setattr(noisy, "_joint_posterior", noiseless)
    monkeypatch.setattr(gp, "cross_covariance", uncorrelated)
    val = torch.from_numpy(sc.scores(x, None, seed=5, n_samples=256))
    rows = sc.baseline[sc.kept_baseline(0)]
    z = sobol_normal_samples(256, 1 + len(rows), 5)
    mu, var = (t.float().double() for t in oracle.posterior(gp.om, x))  # the fp32 moments the scorer is given
    a, b = sc.cfg.obj_scale, sc.cfg.obj_shift
    best_f = float((a * no.joint_posterior_f64(gp, rows)[0] + b).max())
    acq = oracle.AcqSpec(kind="qEI", best_f=best_f, obj_scale=a, obj_shift=b)
    ref = oracle.reference_path.acq_from_moments(acq, mu, var, z[:, -1])
    assert torch.allclose(val, ref, rtol=1e-5, atol=1e-7), float((val - ref).abs().max())


@pytest.mark.parametrize("kind", ["qNEI", "qLogNEI"])
def test_joint_value_of_a_q_batch_matches_brute_force(f64_engine, kind):
    w, gp, sc, pend, _, x = _setup(kind, 2, 0)
    c = sc.cfg
    for q in (1, 2, 4):
        batch = x[:q]
        v = sc.joint_value(batch, pend, seed=4, n_samples=64)
        nc = sc.n_conditioning(2 + q - 1)
        z = sobol_normal_samples(64, 1 + nc, 4).numpy()
        kept = sc.baseline[sc.kept_baseline(2 + q - 1)]
        rows = np.concatenate([kept, pend, batch[1:]])
        ref = float(no.nei_full_joint(gp.om, rows, len(kept) + 2, batch[:1], z, kind == "qLogNEI", c.obj_scale,
                                      c.obj_shift, c.tau_relu, c.tau_max)[0])
        assert abs(v - ref) <= 1e-6 * max(1.0, abs(ref)), (q, v, ref)
    own = sc.scores(x[:1], pend, seed=4, n_samples=64)[0]
    assert sc.joint_value(x[:1], pend, seed=4, n_samples=64) == own


def test_joint_value_rejects_more_than_31_conditioning_points(f64_engine):
    w, gp = _stand_in(n=25)
    sc = noisy.NeiScorer(gp, AcqConfig(kind="qNEI"), w.train_x, prune=False)
    with pytest.raises(NotImplementedError, match="at most 31"):
        sc.joint_value(w.candidates[:8], None, seed=0, n_samples=32)
    assert np.isfinite(sc.joint_value(w.candidates[:7], None, seed=0, n_samples=32))


def test_greedy_rounds_add_the_winner_to_the_conditioning_set(f64_engine, monkeypatch):
    from baybe_b200.recommenders import greedy_select

    w, gp, sc, _, _, x = _setup("qLogNEI", 0, 0)
    seen = []
    values = sc.values

    def spy(x_, pend, *a, **k):
        seen.append(0 if pend is None else len(pend))
        return values(x_, pend, *a, **k)

    monkeypatch.setattr(sc, "values", spy)
    chosen, vals = greedy_select(sc, sc.cfg, torch.from_numpy(x), x.shape[1], 3, None, seed=2, n_samples=64)
    assert seen == [0, 1, 2] and len(set(chosen)) == 3
    for r in range(3):  # each round's value is the f64 value of its winner given the earlier winners
        pend = x[chosen[:r]] if r else None
        ref = sc.scores(x, pend, seed=2, n_samples=64)
        assert abs(ref[chosen[r]] - vals[r]) <= 1e-6 * max(1.0, abs(vals[r]))
        ref[chosen[:r]] = -np.inf
        assert int(np.argmax(ref)) == chosen[r]


# ---- argument checks ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _call_nei(lib, **over):
    p = C.c_void_p(1 << 20)
    args = dict(log=1, a=C.c_float(1.0), b=C.c_float(0.0), tau_relu=C.c_float(1e-6), tau_max=C.c_float(1e-2), N=100,
                mu=p, var=p, C=3, cross=p, linv=p, w=p, z=p, S=64, g=p, Q=0, terms=None, keep=None, score=p, key=p,
                offset=0, stream=None)
    args.update(over)
    return lib.bb_nei_score(*args.values())


_BAD_NEI = [
    ("log flag 2", dict(log=2), b"log_nei=2"),
    ("scale not finite", dict(a=C.c_float(math.inf)), b"not finite"),
    ("tau_relu 0", dict(tau_relu=C.c_float(0.0)), b"tau_relu"),
    ("negative offset", dict(offset=-1), b"32-bit key"),
    ("index overflow", dict(N=1 << 32), b"32-bit key"),
    ("n_cond 32", dict(C=32), b"n_cond=32"),
    ("n_cond -1", dict(C=-1), b"n_cond=-1"),
    ("batch above n_cond", dict(Q=4), b"n_batch=4"),
    ("S = 0", dict(S=0), b"S=0"),
    ("S = 1025", dict(S=1025), b"S=1025"),
    ("null key", dict(key=None), b"null best key"),
    ("null mu", dict(mu=None), b"null buffer"),
    ("null incumbents", dict(g=None), b"null buffer"),
    ("conditioning without w", dict(w=None), b"need cross, linv and w"),
    ("batch without terms", dict(Q=2), b"need their terms"),
]


@pytest.mark.parametrize("case,over,msg", _BAD_NEI, ids=[c for c, *_ in _BAD_NEI])
def test_bb_nei_score_rejects_bad_arguments_before_any_cuda_call(lib, case, over, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    assert _call_nei(lib, **over) == _lib.BB_ERR_INVALID
    assert msg in lib.bb_last_error()


def test_bb_nei_score_accepts_an_empty_candidate_set(lib):
    assert _call_nei(lib, N=0, mu=None, var=None, g=None) == 0


def _call_joint(lib, model, **over):
    m = model
    p = C.c_void_p(1 << 20)
    args = dict(m=C.byref(m), x=p, R=10, mu=p, cov=p, beta=None, ws=p, ws_doubles=10 * (m.n_pad + m.d), stream=None)
    args.update(over)
    return lib.bb_joint_posterior(*args.values())


_BAD_JOINT = [
    ("null model", dict(m=None), "invalid", b"null model"),
    ("ABI mismatch", dict(abi=99), "invalid", b"ABI mismatch"),
    ("R = 0", dict(R=0), "invalid", b"R=0"),
    ("R above n_pad", dict(R=65), "invalid", b"R=65"),
    ("null rows", dict(x=None), "invalid", b"null argument"),
    ("null covariance", dict(cov=None), "invalid", b"null argument"),
    ("small workspace", dict(ws_doubles=10 * 84 - 1), "workspace", b"workspace of 839 doubles"),
]


@pytest.mark.parametrize("case,over,status,msg", _BAD_JOINT, ids=[c for c, *_ in _BAD_JOINT])
def test_bb_joint_posterior_rejects_bad_arguments_before_any_cuda_call(lib, case, over, status, msg):
    from baybe_b200 import _lib
    from tests.test_abi import _fake_model

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    m = _fake_model(False, 1)  # n = n_pad = 64, d = 20
    m.abi_version = over.pop("abi", m.abi_version)
    rc = _call_joint(lib, m, **over)
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "workspace": _lib.BB_ERR_WORKSPACE}[status]
    assert msg in lib.bb_last_error()


def test_nei_kinds_stay_off_the_fused_kernels():
    from baybe_b200.acquisition import convert_acqf, qLogNoisyExpectedImprovement

    spec = convert_acqf("qLogNEI")
    assert isinstance(spec, qLogNoisyExpectedImprovement) and spec.prune_baseline and spec.supports_pending_experiments
    for kind in ("qNEI", "qLogNEI"):
        cfg = AcqConfig(kind=kind)
        assert cfg.is_mc
        with pytest.raises(NotImplementedError):
            cfg.to_c()


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

    monkeypatch.setattr(surrogates, "DeviceGP", no.StandInGP)
    return baybe_plugin


def noisy_campaign(plugin, acqf, objective=None):
    """Shared by the CPU and GPU Campaign tests: the 216-row space of tests/test_mo.py with one noisy target."""
    from baybe import Campaign
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate
    from tests.test_mo import pareto_campaign

    _, space = pareto_campaign(plugin, None)
    d = len(space.comp_rep_columns)
    hyper = {"lengthscale": np.full(d, 0.9), "noise": 5e-2, "mean_const": 0.0}
    rec = plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hyper),
                                        acquisition_function=acqf, n_mc_samples=128)
    objective = objective or SingleTargetObjective(NumericalTarget("yield"))
    return Campaign(space, objective, rec, allow_recommending_already_measured=False), space


def check_noisy_flow(camp, space, rng, tol):
    """recommend -> add_measurements -> recommend; the recommendation is the arg-max of acquisition_values, the
    single-row joint value is its own value, pending experiments are conditioned on."""
    from tests.test_mo import measure

    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, rng, ("yield",)))
    rec = camp.recommend(batch_size=3)
    assert len(rec) == 3 and rec.index.is_unique and not set(rec.index) & set(seed_rows.index)
    camp.add_measurements(measure(rec, rng, ("yield",)))
    torch.manual_seed(11)
    r1 = camp.recommend(batch_size=1)

    def greedy_seed():
        # recommend draws the acquisition callable's sampler seed, then the greedy loop's; the diagnostics draw one
        torch.manual_seed(11)
        torch.randint(0, 1_000_000, (1,))

    greedy_seed()
    vals = camp.acquisition_values(space.discrete.exp_rep)
    remaining = vals.drop(index=list(seed_rows.index) + list(rec.index))
    assert np.isfinite(vals.to_numpy()).all()
    assert float(vals.loc[r1.index[0]]) >= float(remaining.max()) - tol * max(1.0, abs(float(remaining.max())))
    greedy_seed()
    jv = camp.joint_acquisition_value(r1)
    assert abs(jv - float(vals.loc[r1.index[0]])) <= tol * max(1.0, abs(jv))
    torch.manual_seed(12)
    with_pending = camp.acquisition_values(space.discrete.exp_rep.head(20), pending_experiments=r1)
    torch.manual_seed(12)
    assert not np.allclose(with_pending.to_numpy(), camp.acquisition_values(space.discrete.exp_rep.head(20)))
    rec3 = camp.recommend(batch_size=3, pending_experiments=r1)
    assert len(rec3) == 3 and r1.index[0] not in rec3.index
    return vals


@pytest.mark.parametrize("kind", ["qNEI", "qLogNEI"])
def test_noisy_campaign_on_the_stand_in_engine(bb, kind):
    from baybe.acquisition import acqfs

    acqf = {"qNEI": acqfs.qNoisyExpectedImprovement, "qLogNEI": acqfs.qLogNoisyExpectedImprovement}[kind]
    camp, space = noisy_campaign(bb, acqf())
    check_noisy_flow(camp, space, np.random.default_rng(0), tol=0.0)
    assert isinstance(camp.recommender._scorer, noisy.NeiScorer)


def test_prune_baseline_false_through_the_campaign(bb):
    from baybe.acquisition import acqfs

    from tests.test_mo import measure

    camp, space = noisy_campaign(bb, acqfs.qLogNoisyExpectedImprovement(prune_baseline=False))
    camp.add_measurements(measure(space.discrete.exp_rep.sample(12, random_state=1), np.random.default_rng(0),
                                  ("yield",)))
    assert len(camp.recommend(batch_size=2)) == 2
    camp.add_measurements(measure(space.discrete.exp_rep.sample(25, random_state=2), np.random.default_rng(1),
                                  ("yield",)))
    with pytest.raises(NotImplementedError, match="prune_baseline=False"):
        camp.recommend(batch_size=1)


def test_noisy_subset_constraint_on_the_stand_in_engine(bb, monkeypatch):
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
    rec = bb.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp), n_mc_samples=128,
                                    acquisition_function=acqfs.qNoisyExpectedImprovement())
    camp = Campaign(space, SingleTargetObjective(NumericalTarget("t1")), rec)
    rows = space.discrete.exp_rep.sample(8, random_state=0)
    meas = rows.copy()
    shift = rows["cat"].map({"p": 0.0, "q": 0.3, "r": -0.2}).astype(float)
    meas["t1"] = rows["x"] - (rows["y"] - 0.5) ** 2 + shift + np.random.default_rng(5).normal(0, 0.05, len(rows))
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


def test_noisy_rejections(bb):
    from baybe import Campaign
    from baybe.acquisition import acqfs
    from baybe.exceptions import IncompatibleAcquisitionFunctionError
    from baybe.objectives import SingleTargetObjective
    from baybe.parameters import NumericalContinuousParameter, NumericalDiscreteParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget

    from baybe_b200.surrogates import GaussianProcessSurrogate
    from tests.test_mo import measure

    # qLogNEI on a hybrid space
    space = SearchSpace.from_product([NumericalDiscreteParameter("a", values=[0.0, 0.5, 1.0]),
                                      NumericalContinuousParameter("b", bounds=(0.0, 1.0))])
    hp = {"lengthscale": np.full(2, 0.9), "noise": 5e-3, "mean_const": 0.0}
    camp = Campaign(space, SingleTargetObjective(NumericalTarget("t")), bb.B200BotorchRecommender(
        surrogate_model=GaussianProcessSurrogate(hyperparameters=hp),
        acquisition_function=acqfs.qLogNoisyExpectedImprovement()))
    meas = space.discrete.exp_rep.sample(3, random_state=0, replace=True).reset_index(drop=True)
    meas["b"] = [0.2, 0.5, 0.9]
    meas["t"] = [0.1, 0.4, 0.3]
    camp.add_measurements(meas)
    with pytest.raises(IncompatibleAcquisitionFunctionError):
        camp.recommend(batch_size=1)
    # a non-affine single target
    camp, space = noisy_campaign(bb, acqfs.qNoisyExpectedImprovement(), SingleTargetObjective(
        NumericalTarget.match_triangular("yield", cutoffs=(50.0, 60.0))))
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), np.random.default_rng(2),
                                  ("yield",)))
    with pytest.raises(NotImplementedError, match="affine in one modelled target"):
        camp.recommend(batch_size=1)


@pytest.mark.parametrize("kind", ["qNEI", "qLogNEI"])
def test_desirability_objectives_with_noisy_ei(bb, kind):
    """Desirability computed on several models is rejected with a message naming the fix (recommend and the
    diagnostics alike, before any model is fitted); applied as a pre-transformation it is one affine target."""
    from baybe.acquisition import acqfs
    from baybe.objectives import DesirabilityObjective
    from baybe.targets import NumericalTarget

    from tests.test_mo import measure

    acqf = {"qNEI": acqfs.qNoisyExpectedImprovement, "qLogNEI": acqfs.qLogNoisyExpectedImprovement}[kind]
    targets = [NumericalTarget("yield").clamp(45.0, 60.0).normalize(),
               NumericalTarget("cost", minimize=True).clamp(4.0, 7.0).normalize()]
    rows = measure(_noisy_space_rows(bb), np.random.default_rng(4))
    camp, space = noisy_campaign(bb, acqf(), DesirabilityObjective(targets))
    camp.add_measurements(rows)
    for call in (lambda: camp.recommend(batch_size=2), lambda: camp.acquisition_values(space.discrete.exp_rep.head(5)),
                 lambda: camp.joint_acquisition_value(space.discrete.exp_rep.head(2))):
        with pytest.raises(NotImplementedError, match="several models: use as_pre_transformation=True"):
            call()
    camp, space = noisy_campaign(bb, acqf(), DesirabilityObjective(targets, as_pre_transformation=True))
    camp.add_measurements(rows)
    rec = camp.recommend(batch_size=2)
    assert len(rec) == 2 and isinstance(camp.recommender._scorer, noisy.NeiScorer)


def _noisy_space_rows(plugin):
    _, space = noisy_campaign(plugin, None)
    return space.discrete.exp_rep.sample(12, random_state=1)
