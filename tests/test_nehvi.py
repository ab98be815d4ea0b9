"""CPU tests of qNEHVI on discrete spaces: the baseline pruning against a brute-force restatement, the conditional value
against the definition mean_s[hv(F_s u O_s u {y_s}) - hv(F_s)] from the full joint Cholesky of [C; x] and a brute-force
hypervolume, metamorphic checks (qEHVI limit, affine rescaling, flipped targets), the argument checks of
``bb_hvi_decompose`` and the Campaign glue on a float64 stand-in engine."""
from __future__ import annotations

import ctypes as C
import dataclasses
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import multiobjective as mo
from baybe_b200 import nehvi, noisy
from baybe_b200.engine import AcqConfig, sobol_normal_samples
from baybe_b200.synthetic import numeric_grid_workload
from tests import mo_oracle
from tests import parego_oracle as po
from tests.test_mo import _hvi_score_f64

ROOT = Path(__file__).resolve().parents[1]
CFG = AcqConfig(kind="qNEHVI")


def decompose_f64(points, ref, device=None):
    """Float64 stand-in of ``nehvi._hvi_decompose``: ``box_decomposition`` of every sample's points, padded."""
    pts = np.asarray(points, dtype=np.float64)
    decs = [mo.box_decomposition(p, ref) for p in pts]
    M = pts.shape[2]
    width = max(1, max(len(lo) for lo, _, _ in decs))
    lower, upper = np.zeros((len(decs), width, M)), np.zeros((len(decs), width, M))
    for k, (lo, up, _) in enumerate(decs):
        lower[k, :len(lo)], upper[k, :len(up)] = lo, up
    return (torch.from_numpy(lower), torch.from_numpy(upper),
            torch.tensor([len(lo) for lo, _, _ in decs], dtype=torch.int32),
            torch.tensor([hv for _, _, hv in decs], dtype=torch.float64))


@pytest.fixture()
def f64_engine(monkeypatch):
    monkeypatch.setattr(noisy, "_joint_posterior", po.joint_posterior_f64)
    monkeypatch.setattr(nehvi, "_hvi_decompose", decompose_f64)
    monkeypatch.setattr(nehvi, "_hvi_score", _hvi_score_f64)
    monkeypatch.setattr(mo, "_hvi_score", _hvi_score_f64)


def _scorer(M=2, n=8, seed=0, N=200, d=4, prune=False, noise=1e-2, scales=None, shifts=None, ref=None, **kw):
    w = numeric_grid_workload(N=N, d=d, n=n, seed=seed)
    gps = po.stand_in_models(w, M, noise=noise, seed=seed)
    a = np.array(scales if scales is not None else [1.0, -1.0] * (M // 2) + [1.0] * (M % 2))
    b = np.array(shifts if shifts is not None else np.linspace(0.0, 0.5, M))
    if ref is None:
        ref = mo.compute_ref_point(np.stack([g.train_y for g in gps], 1) * a + b)
    return w, gps, nehvi.NehviScorer(gps, dataclasses.replace(CFG, **kw), a, b, ref, w.train_x, prune=prune)


def _unmeasured(w, k, seed):
    X = w.candidates  # a measured candidate would make the joint covariance of [C; x] singular
    X = X[np.abs(X[:, None, :] - w.train_x[None]).sum(-1).min(1) > 1e-9]
    return X[np.random.default_rng(seed).choice(len(X), k, replace=False)]


# ---- pruning -----------------------------------------------------------------------------------------------------------------
def _brute_pareto_counts(Y, ref):
    """Per row, in how many samples of Y [samples, n, M] no other row dominates it and it is strictly above ref."""
    S, n, _ = Y.shape
    counts = np.zeros(n, dtype=np.int64)
    for s in range(S):
        for i in range(n):
            dominated = any((Y[s, j] >= Y[s, i]).all() and (Y[s, j] > Y[s, i]).any() for j in range(n) if j != i)
            counts[i] += (not dominated) and bool((Y[s, i] > ref).all())
    return counts


@pytest.mark.parametrize("M", [2, 3])
def test_pruning_keeps_the_rows_on_some_sampled_front(f64_engine, M):
    w, gps, _ = _scorer(M=M, n=10, seed=M)
    X = w.train_x
    a = np.array([1.0, -1.0, 1.0][:M])
    b = np.zeros(M)
    mu0 = np.stack([po.joint_posterior_f64(g, X)[0] for g in gps], 1) * a + b
    ref = np.median(mu0, axis=0)  # a reference point in the middle of the cloud: the filter matters
    sc = nehvi.NehviScorer(gps, CFG, a, b, ref, X, prune=True, prune_seed=4)
    n = len(X)
    z = sobol_normal_samples(noisy.PRUNE_SAMPLES, M * n, 4).numpy()
    Y = np.empty((noisy.PRUNE_SAMPLES, n, M))
    for m, g in enumerate(gps):
        mu, cov = oracle.posterior_joint(g.om, X)
        L = mo._psd_cholesky(0.5 * (cov.numpy() + cov.numpy().T))
        Y[:, :, m] = a[m] * (mu.numpy()[None] + z[:, m * n:(m + 1) * n] @ L.T) + b[m]
    counts_sc = np.zeros(n, dtype=np.int64)
    counts_sc[sc.winners] = sc.counts
    assert np.array_equal(counts_sc, _brute_pareto_counts(Y, ref))  # all 2048 samples, across every chunk boundary
    assert 0 < len(sc.winners) < n
    for n_other in (0, 31 - len(sc.winners) + 2):
        cap = 31 - n_other
        order = sorted(range(len(sc.winners)), key=lambda k: -sc.counts[k])  # stable: ties keep index order
        expect = sorted(sc.winners[order[:cap]]) if len(sc.winners) > cap else list(sc.winners)
        assert list(sc.kept_baseline(n_other)) == [int(v) for v in expect]
        assert sc.n_dropped == len(sc.winners) - len(expect)


def test_pareto_mask_keeps_duplicates_and_applies_the_reference_point():
    Y = np.array([[[1.0, 2.0], [1.0, 2.0], [0.0, 1.0], [2.0, 0.5], [3.0, 0.0]]])
    assert nehvi.pareto_mask(Y, np.array([0.0, 0.0])).tolist() == [[True, True, False, True, False]]
    assert nehvi.pareto_mask(Y, np.array([-1.0, -1.0])).tolist() == [[True, True, False, True, True]]


def test_prune_baseline_false_conditions_on_every_row_up_to_the_limit(f64_engine):
    w, gps, sc = _scorer(M=2, n=29, prune=False)
    assert list(sc.kept_baseline(2)) == list(range(29)) and sc.n_dropped == 0
    with pytest.raises(NotImplementedError, match="prune_baseline=False.*at most 31"):
        sc.kept_baseline(3)


# ---- the value ----------------------------------------------------------------------------------------------------------------
def _definition(sc, gps, rows, n_front, x, z):
    """mean_s[hv(F_s u O_s u {y_s}) - hv(F_s)] for every row of x, from the joint Cholesky of [rows; x_i] per target
    with the same base samples and the brute-force hypervolume of tests/mo_oracle.py."""
    nc, M = len(rows), sc.M
    out = np.empty(len(x))
    for i in range(len(x)):
        Y = np.empty((z.shape[0], nc + 1, M))
        for m, g in enumerate(gps):
            mean, cov = oracle.posterior_joint(g.om, np.concatenate([rows, x[i:i + 1]]))
            L = torch.linalg.cholesky(cov).numpy()
            Y[:, :, m] = sc.a[m] * (mean.numpy()[None] + z[:, m * (nc + 1):(m + 1) * (nc + 1)] @ L.T) + sc.b[m]
        out[i] = np.mean([mo_oracle.hv(Y[s], sc.ref) - mo_oracle.hv(Y[s, :n_front], sc.ref) for s in range(len(Y))])
    return out


def _engine_form(sc, gps, pend, batch, x, z):
    """The scorer's own conditioning, the candidate sampled conditionally on C in float64, the improvement over each
    sample's decomposition of F_s u O_s, plus the batch points' mean_s(hv(F_s u O_s) - hv(F_s))."""
    rows, linv, w, o, _ = sc.conditioning(pend, batch, z)
    nc, M = len(rows), sc.M
    Q = 0 if batch is None else len(batch)
    Y = np.empty((z.shape[0], len(x), M))
    for m, g in enumerate(gps):
        mu, var = (t.numpy() for t in oracle.posterior(g.om, x))
        zx = z[:, m * (nc + 1) + nc]
        if nc:
            _, cov = oracle.posterior_joint(g.om, np.concatenate([rows, x]))
            c = cov.numpy()[nc:, :nc]
            r = c @ linv[m].T
            sd = np.sqrt(np.maximum(var - (r * r).sum(1), 0.0))
            Y[:, :, m] = mu[None] + w[m] @ c.T + sd[None] * zx[:, None]
        else:
            Y[:, :, m] = mu[None] + np.sqrt(var)[None] * zx[:, None]
    Y = Y * sc.a + sc.b
    val, gain = np.zeros(len(x)), []
    for s in range(z.shape[0]):
        lo, up, hv = mo.box_decomposition(o[s], sc.ref)
        val += mo.hvi_hard(lo, up, Y[s]) / z.shape[0]
        gain.append(hv - mo.box_decomposition(o[s, : nc - Q], sc.ref)[2])
    return val + (np.mean(gain) if Q else 0.0), rows


@pytest.mark.parametrize("M", [2, 3, 4])
@pytest.mark.parametrize("P,Q", [(0, 0), (2, 0), (0, 2), (2, 1)])
def test_conditional_value_equals_the_definition(f64_engine, M, P, Q):
    w, gps, sc = _scorer(M=M, n=5, seed=M + P)
    X = _unmeasured(w, P + Q + 4, 10 + M)
    pend, batch, x = (X[:P] if P else None), (X[P:P + Q] if Q else None), X[P + Q:]
    nc = sc.n_conditioning(P + Q)
    z = sobol_normal_samples(16, M * (1 + nc), 7).numpy()
    val, rows = _engine_form(sc, gps, pend, batch, x, z)
    ref = _definition(sc, gps, rows, nc - Q, x, z)
    assert np.allclose(val, ref, rtol=1e-10, atol=1e-10), np.abs(val - ref).max()
    # the scorer through both stand-in seams (fp32 samples and moments in the plumbing)
    s = sc.scores(x, pend, seed=7, n_samples=16, batch=batch)
    assert np.allclose(s, ref, rtol=1e-4, atol=1e-6), np.abs(s - ref).max()


def test_without_any_conditioning_point_the_front_is_empty(f64_engine):
    """A reference point above every measured row keeps no baseline row: C is empty and the value is the expected
    hypervolume of the candidate alone."""
    w, gps, sc0 = _scorer(M=2, n=6)
    sc = nehvi.NehviScorer(gps, CFG, sc0.a, sc0.b, sc0.ref + 50.0, w.train_x, prune=True)
    assert len(sc.winners) == 0 and sc.n_conditioning(0) == 0
    x = _unmeasured(w, 5, 3)
    z = sc.base_samples(32, 0, seed=2).numpy()
    val, _ = _engine_form(sc, gps, None, None, x, z)
    assert np.allclose(sc.scores(x, None, seed=2, n_samples=32), val, rtol=1e-4, atol=1e-8)


def test_noise_free_limit_is_qehvi(f64_engine):
    """With a nearly noise-free model the sampled front collapses to the posterior-mean front and qNEHVI (no pending
    points) equals qEHVI with the same candidate base samples.  The models' noise is 1e-4 (the floor), so the sampled
    front moves by about 1e-2 posterior standard deviations: stated tolerance 2e-2 relative to the largest value."""
    w, gps, sc = _scorer(M=2, n=12, noise=1e-4, prune=True)
    x = _unmeasured(w, 60, 5)
    front = np.stack([po.joint_posterior_f64(g, w.train_x)[0] for g in gps], 1) * sc.a + sc.b
    ehvi = mo.HviScorer(gps, AcqConfig(kind="qEHVI"), sc.a, sc.b, sc.ref, front)
    nc = sc.n_conditioning(0)
    z = sobol_normal_samples(256, 2 * (1 + nc), 3)
    zc = torch.stack([z[:, m * (nc + 1) + nc] for m in range(2)], 1)  # the candidate's columns
    v_nehvi = sc.values(x, None, z)[0].double().numpy()
    v_ehvi = ehvi.values(x, None, zc)[0].double().numpy()
    assert np.abs(v_nehvi - v_ehvi).max() <= 2e-2 * np.abs(v_ehvi).max()
    assert int(np.argmax(v_nehvi)) == int(np.argmax(v_ehvi))


def _rebuilt(w, gps, sc, m, y_map, scale_m=None, ref_m=None):
    new = list(gps)
    new[m] = po.StandInGP(**dataclasses.replace(w, train_y=y_map(gps[m].train_y), noise=np.array([1e-2])).gp_kwargs())
    a, ref = sc.a.copy(), sc.ref.copy()
    if scale_m is not None:
        a[m] = scale_m
    if ref_m is not None:
        ref[m] = ref_m
    return nehvi.NehviScorer(new, sc.cfg, a, sc.b, ref, w.train_x, prune=sc.prune)


def test_rescaled_target_scales_values_and_keeps_the_recommendation(f64_engine):
    """Standardize makes the posterior of 3y + 5 the affine image of y's; with the reference point mapped the same
    way every box and every hypervolume stretch by 3 along that target."""
    w, gps, sc = _scorer(M=3, n=10, scales=[1.0, 1.0, 1.0], shifts=[0.0, 0.0, 0.0], prune=True)
    x = _unmeasured(w, 152, 4)
    pend, x = x[:2], x[2:]  # a candidate at a pending point would leave only fp32 rounding in its variance
    scaled = _rebuilt(w, gps, sc, 1, lambda y: 3.0 * y + 5.0, ref_m=3.0 * sc.ref[1] + 5.0)
    assert list(scaled.winners) == list(sc.winners)
    for p in (None, pend):
        ref = sc.scores(x, p, seed=3, n_samples=128)
        new = scaled.scores(x, p, seed=3, n_samples=128)
        assert np.allclose(new, 3.0 * ref, rtol=1e-4, atol=1e-6 * np.abs(ref).max())
        assert int(np.argmax(new)) == int(np.argmax(ref))


def test_flipped_target_keeps_the_recommendation(f64_engine):
    """Negating a target's measurements and flipping it to minimize=True leaves its orientation o = y in distribution:
    drawn with that target's base samples negated, every sample path is the same, so the values are the same up to
    rounding."""
    w, gps, sc = _scorer(M=2, n=10, scales=[1.0, 1.0], shifts=[0.0, 0.0])
    x = _unmeasured(w, 152, 6)
    pend2, x = x[:2], x[2:]
    flipped = _rebuilt(w, gps, sc, 1, lambda y: -y, scale_m=-1.0)
    for P in (0, 2):
        z = sc.base_samples(128, P, seed=5)
        k = z.shape[1] // 2
        zf = torch.cat([z[:, :k], -z[:, k:]], 1)  # target 1's block negated
        pend = pend2 if P else None
        ref = sc.values(x, pend, z)[0].double().numpy()
        new = flipped.values(x, pend, zf)[0].double().numpy()
        assert np.allclose(new, ref, rtol=1e-4, atol=1e-6 * np.abs(ref).max())
        assert int(np.argmax(new)) == int(np.argmax(ref))


def test_greedy_rounds_add_the_winner_to_the_conditioning_set(f64_engine):
    from baybe_b200.recommenders import greedy_select

    w, gps, sc = _scorer(M=2, n=8)
    x = _unmeasured(w, 60, 1)
    chosen, vals = greedy_select(sc, sc.cfg, torch.from_numpy(x), x.shape[1], 3, None, seed=2, n_samples=32)
    assert len(set(chosen)) == 3
    for r in range(3):
        ref = sc.scores(x, x[chosen[:r]] if r else None, seed=2, n_samples=32)
        assert abs(ref[chosen[r]] - vals[r]) <= 1e-6 * max(1.0, abs(vals[r]))
        ref[chosen[:r]] = -np.inf
        assert int(np.argmax(ref)) == chosen[r]


def test_scorer_rejects_target_counts_outside_2_to_4(f64_engine):
    w = numeric_grid_workload(N=50, d=3, n=6, seed=0)
    for M in (1, 5):
        gps = po.stand_in_models(w, M)
        with pytest.raises(Exception, match="2 to 4 targets"):
            nehvi.NehviScorer(gps, CFG, np.ones(M), np.zeros(M), np.zeros(M), w.train_x)


def test_nehvi_kind_stays_off_the_fused_kernels():
    from baybe_b200.acquisition import convert_acqf, qNoisyExpectedHypervolumeImprovement

    spec = convert_acqf("qNEHVI")
    assert isinstance(spec, qNoisyExpectedHypervolumeImprovement) and spec.prune_baseline
    assert spec.supports_multi_output and spec.supports_batching and spec.supports_pending_experiments
    assert convert_acqf("qNoisyExpectedHypervolumeImprovement").reference_point is None
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
    args = dict(M=3, ref=(C.c_double * 4)(0.0, 0.0, 0.0, 0.0), S=64, n=10, pts=p, n_pts=None, stride=1024, lo=p,
                up=p, cells=p, hv=p, stream=None)
    args.update(over)
    return lib.bb_hvi_decompose(*args.values())


_BAD = [
    ("one target", dict(M=1), "unsupported", b"n_targets=1"),
    ("five targets", dict(M=5), "unsupported", b"n_targets=5"),
    ("null ref", dict(ref=None), "invalid", b"null reference"),
    ("ref not finite", dict(ref=(C.c_double * 4)(0.0, float("nan"), 0.0, 0.0)), "invalid", b"target 1 not finite"),
    ("S = 0", dict(S=0), "invalid", b"S=0"),
    ("S = 1025", dict(S=1025), "invalid", b"S=1025"),
    ("n = 32", dict(n=32), "invalid", b"n=32"),
    ("n = -1", dict(n=-1), "invalid", b"n=-1"),
    ("stride 0", dict(stride=0), "unsupported", b"cell_stride=0"),
    ("stride 1025", dict(stride=1025), "unsupported", b"cell_stride=1025"),
    ("null hv", dict(hv=None), "invalid", b"null output"),
    ("null points", dict(pts=None), "invalid", b"null points"),
]


@pytest.mark.parametrize("case,over,status,msg", _BAD, ids=[c for c, *_ in _BAD])
def test_bb_hvi_decompose_rejects_bad_arguments_before_any_cuda_call(lib, case, over, status, msg):
    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    assert _call(lib, **over) == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status]
    assert msg in lib.bb_last_error()


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


NAMES = ("yield", "cost", "purity", "speed")


def check_nehvi_flow(plugin, monkeypatch, n_targets, tol):
    """Shared by the CPU and GPU Campaign tests: a Pareto campaign of `n_targets` targets with qNEHVI through
    recommend (a greedy batch of 3, then one row, then pending experiments), ``acquisition_values`` (its arg-max is the
    recommended row under the same seed and sample count) and ``joint_acquisition_value``."""
    from baybe.acquisition.acqfs import qNoisyExpectedHypervolumeImprovement
    from baybe.targets import NumericalTarget

    from baybe_b200 import baybe_plugin, recommenders
    from baybe_b200.engine import DEFAULT_MC_SAMPLES
    from tests.test_mo import measure, pareto_campaign

    names = NAMES[:n_targets]
    targets = [NumericalTarget(n, minimize=(n == "cost")) for n in names]
    rng = np.random.default_rng(0)
    # one sampler seed and sample count for every draw, so that recommend and the diagnostics score alike
    for mod in (recommenders, baybe_plugin):
        monkeypatch.setattr(mod, "_draw_sampler_seed", lambda: 77)
    camp, space = pareto_campaign(plugin, qNoisyExpectedHypervolumeImprovement(), targets=targets)
    camp.recommender.n_mc_samples = DEFAULT_MC_SAMPLES
    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, np.random.default_rng(0), names))
    rec = camp.recommend(batch_size=3)
    assert len(rec) == 3 and rec.index.is_unique and not set(rec.index) & set(seed_rows.index)
    scorer = camp.recommender._scorer
    assert isinstance(scorer, nehvi.NehviScorer) and scorer.M == n_targets and len(scorer.winners) > 0
    camp.add_measurements(measure(rec, rng, names))
    r1 = camp.recommend(batch_size=1)
    vals = camp.acquisition_values(space.discrete.exp_rep)
    assert np.isfinite(vals.to_numpy()).all() and (vals.to_numpy() >= 0).all()
    remaining = vals.drop(index=list(seed_rows.index) + list(rec.index))
    assert float(vals.loc[r1.index[0]]) >= float(remaining.max()) - tol * max(1.0, abs(float(remaining.max())))
    jv = camp.joint_acquisition_value(r1)
    assert abs(jv - float(vals.loc[r1.index[0]])) <= tol * max(1.0, abs(jv))
    two = space.discrete.exp_rep.loc[[r1.index[0], remaining.index[0]]]
    assert np.isfinite(camp.joint_acquisition_value(two))
    with_pending = camp.acquisition_values(space.discrete.exp_rep.head(20), pending_experiments=r1)
    assert not np.allclose(with_pending.to_numpy(), camp.acquisition_values(space.discrete.exp_rep.head(20)))
    rec3 = camp.recommend(batch_size=3, pending_experiments=r1)
    assert len(rec3) == 3 and r1.index[0] not in rec3.index
    return camp


@pytest.mark.parametrize("n_targets", [2, 3])
def test_nehvi_campaign_on_the_stand_in_engine(bb, monkeypatch, n_targets):
    check_nehvi_flow(bb, monkeypatch, n_targets, tol=1e-6)


def test_nehvi_subset_constraint_on_the_stand_in_engine(bb, monkeypatch):
    from baybe.acquisition.acqfs import qNoisyExpectedHypervolumeImprovement

    from tests.test_mo import check_subset_batch_wins

    check_subset_batch_wins(bb, monkeypatch, np.random.default_rng(5), qNoisyExpectedHypervolumeImprovement())


def test_nehvi_rejections(bb):
    from baybe import Campaign
    from baybe.acquisition.acqfs import qNoisyExpectedHypervolumeImprovement as qNEHVI
    from baybe.exceptions import IncompatibleAcquisitionFunctionError
    from baybe.objectives import ParetoObjective, SingleTargetObjective
    from baybe.parameters import NumericalContinuousParameter, NumericalDiscreteParameter
    from baybe.searchspace import SearchSpace
    from baybe.targets import NumericalTarget
    from baybe.transformations import ExponentialTransformation

    from baybe_b200.surrogates import GaussianProcessSurrogate
    from tests.test_mo import measure, pareto_campaign

    rng = np.random.default_rng(2)
    camp, space = pareto_campaign(bb, qNEHVI())
    hp = {"lengthscale": np.full(len(space.comp_rep_columns), 0.9), "noise": 5e-3, "mean_const": 0.0}
    single = Campaign(space, SingleTargetObjective(NumericalTarget("yield")), bb.B200BotorchRecommender(
        surrogate_model=GaussianProcessSurrogate(hyperparameters=hp)))
    single.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng, ("yield",)))
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="multi-output"):
        single.acquisition_values(space.discrete.exp_rep.head(5), acquisition_function=qNEHVI())
    names = ("yield", "cost", "purity", "speed", "waste")
    camp, space = pareto_campaign(bb, qNEHVI(), targets=[NumericalTarget(n) for n in names])
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng, names))
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="2 to 4 targets"):
        camp.recommend(batch_size=1)
    camp, space = pareto_campaign(bb, qNEHVI(), targets=[
        NumericalTarget("yield"), NumericalTarget("cost", transformation=ExponentialTransformation(), minimize=True)])
    camp.add_measurements(measure(space.discrete.exp_rep.sample(10, random_state=3), rng))
    with pytest.raises(NotImplementedError, match="not affine"):
        camp.recommend(batch_size=1)
    space = SearchSpace.from_product([NumericalDiscreteParameter("a", values=[0.0, 0.5, 1.0]),
                                      NumericalContinuousParameter("b", bounds=(0.0, 1.0))])
    hp = {"lengthscale": np.full(2, 0.9), "noise": 5e-3, "mean_const": 0.0}
    camp = Campaign(space, ParetoObjective([NumericalTarget("t1"), NumericalTarget("t2", minimize=True)]),
                    bb.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp),
                                              acquisition_function=qNEHVI()))
    meas = space.discrete.exp_rep.sample(3, random_state=0, replace=True).reset_index(drop=True)
    meas["b"], meas["t1"], meas["t2"] = [0.2, 0.5, 0.9], [0.1, 0.4, 0.3], [1.0, 0.2, 0.5]
    camp.add_measurements(meas)
    with pytest.raises(IncompatibleAcquisitionFunctionError, match="discrete search spaces only"):
        camp.recommend(batch_size=1)
