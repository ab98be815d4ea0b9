"""CPU tests of the oracle itself.  PARITY UNPINNED: the reference holds no golden vectors for this
path and botorch/gpytorch cannot be installed offline, so the oracle is cross-checked against
independent implementations (scikit-learn GP posterior, scipy normal distribution, closed forms,
Monte-Carlo vs analytic consistency) and against the committed fixtures in tests/golden/."""
from __future__ import annotations

import json
import math
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy.stats import norm

import oracle
from baybe_b200.synthetic import mixed_small_workload, numeric_grid_workload, task_workload
from tests.helpers import oracle_model

GOLDEN = Path(__file__).parent / "golden"


def _sk_kernel(family, ls):
    from sklearn.gaussian_process.kernels import RBF, Matern

    if family == "rbf":
        return RBF(length_scale=ls, length_scale_bounds="fixed")
    nu = {"matern12": 0.5, "matern32": 1.5, "matern52": 2.5}[family]
    return Matern(length_scale=ls, length_scale_bounds="fixed", nu=nu)


@pytest.mark.parametrize("family", ["matern12", "matern32", "matern52", "rbf"])
def test_posterior_matches_sklearn(family):
    from sklearn.gaussian_process import GaussianProcessRegressor
    from sklearn.gaussian_process.kernels import ConstantKernel

    w = numeric_grid_workload(N=300, d=6, n=40, family=family, lengthscale=np.linspace(0.3, 1.1, 6),
                              outputscale=1.7, noise=2e-3, seed=11)
    om = oracle_model(w)
    mu, var = oracle.posterior(om, w.candidates)
    yt = (w.train_y - w.train_y.mean()) / w.train_y.std(ddof=1)
    gp = GaussianProcessRegressor(ConstantKernel(1.7, "fixed") * _sk_kernel(family, w.lengthscale),
                                  alpha=2e-3, optimizer=None).fit(w.train_x, yt)
    ms, ss = gp.predict(w.candidates, return_std=True)
    s = w.train_y.std(ddof=1)
    # Matern-1/2 is sqrt-singular at r=0: the GEMM-form distance (gpytorch's, restated by the
    # oracle) turns 1e-16 of cancellation into 1e-8 at coincident points; sklearn uses cdist.
    tol = 1e-6 if family == "matern12" else 1e-10
    assert np.abs(mu.numpy() - (w.train_y.mean() + s * ms)).max() < tol
    assert np.abs(var.numpy() - (s * ss) ** 2).max() < tol


def test_closed_form_single_training_point():
    # n=1: mean = c + k/(1+noise) * (y~ - c), var = 1 - k^2/(1+noise), Standardize with n=1 -> std 1
    spec = oracle.KernelSpec("matern52", [0.7], [0])
    om = oracle.build_model(spec, np.array([[0.25]]), np.array([3.0]), np.array([[0.0], [1.0]]),
                            noise=0.01, mean_const=0.2)
    x = np.array([[0.6]])
    r = abs(0.6 - 0.25) / 0.7
    k = (1 + math.sqrt(5) * r + 5 / 3 * r * r) * math.exp(-math.sqrt(5) * r)
    mu, var = oracle.posterior(om, x)
    assert om.y_std == 1.0 and om.y_mean == 3.0
    assert abs(float(mu) - (3.0 + 0.2 + k / 1.01 * (0.0 - 0.2))) < 1e-12
    assert abs(float(var) - (1 - k * k / 1.01)) < 1e-12


def test_normalisation_uses_scaling_bounds_not_data():
    w = mixed_small_workload()
    om = oracle_model(w)
    assert torch.allclose(om.lo, torch.tensor(w.bounds[0]))
    assert float(om.Xn.min()) >= 0.0 and float(om.Xn.max()) <= 1.0
    # degenerate range -> 1 (botorch Normalize), task column untouched
    spec = oracle.KernelSpec("rbf", [1.0, 1.0], [0, 1])
    m = oracle.build_model(spec, np.array([[2.0, 5.0], [3.0, 5.0]]), np.array([0.0, 1.0]),
                           np.array([[2.0, 5.0], [3.0, 5.0]]), noise=1e-2)
    assert float(m.rng[1]) == 1.0


def test_noise_floor_and_jitter():
    spec = oracle.KernelSpec("rbf", [5.0], [0])
    X = np.linspace(0, 1, 30).reshape(-1, 1)
    m = oracle.build_model(spec, X, np.sin(X[:, 0]), np.array([[0.0], [1.0]]), noise=1e-9)
    assert float(m.noise) == oracle.reference_path.MIN_INFERRED_NOISE_LEVEL
    assert torch.isfinite(m.alpha).all()


def test_analytic_acquisition_against_scipy():
    w = numeric_grid_workload(N=400, d=4, n=25, seed=5)
    om = oracle_model(w)
    mu, var = oracle.posterior(om, w.candidates)
    sd = var.sqrt().numpy()
    best = 1.1 * float(mu.max())
    u = (mu.numpy() - best) / sd
    ei = oracle.acq_values(om, oracle.AcqSpec("EI", best_f=best), w.candidates).numpy()
    mid = np.abs(u) < 6  # the plain formula cancels catastrophically further out (LogEI covers it)
    assert np.allclose(ei[mid], (sd * (norm.pdf(u) + u * norm.cdf(u)))[mid], rtol=1e-8, atol=0)
    pi = oracle.acq_values(om, oracle.AcqSpec("PI", best_f=best), w.candidates).numpy()
    assert np.allclose(pi, norm.cdf(u), rtol=1e-10, atol=1e-300)
    ucb = oracle.acq_values(om, oracle.AcqSpec("UCB", beta=0.2), w.candidates).numpy()
    assert np.allclose(ucb, mu.numpy() + math.sqrt(0.2) * sd)
    logei = oracle.acq_values(om, oracle.AcqSpec("LogEI", best_f=best), w.candidates).numpy()
    assert np.allclose(logei[mid], np.log(ei[mid]), rtol=1e-8, atol=1e-8)
    # far left tail stays finite and monotone where plain log(EI) underflows
    far = oracle.reference_path._log_ei_helper(torch.tensor([-50.0, -200.0, -1e5, -1e7], dtype=torch.float64))
    assert torch.isfinite(far).all() and bool((far[:-1] > far[1:]).all())


def test_mc_acquisition_converges_to_analytic():
    w = numeric_grid_workload(N=200, d=4, n=25, seed=6)
    om = oracle_model(w)
    z = oracle.sobol_normal_samples(8192, 1, 3)[:, 0]
    best = oracle.best_f_from_training(om, w.train_x, oracle.AcqSpec("qEI"))
    qei = oracle.acq_values(om, oracle.AcqSpec("qEI", best_f=best), w.candidates, z)
    ei = oracle.acq_values(om, oracle.AcqSpec("EI", best_f=best), w.candidates)
    assert float((qei - ei).abs().max()) < 2e-3 * float(ei.max()) + 1e-6
    qlog = oracle.acq_values(om, oracle.AcqSpec("qLogEI", best_f=best), w.candidates, z)
    big = ei > 1e-3 * ei.max()
    assert float((qlog[big] - ei[big].log()).abs().max()) < 5e-2
    qucb = oracle.acq_values(om, oracle.AcqSpec("qUCB", beta=0.2), w.candidates, z)
    ucb = oracle.acq_values(om, oracle.AcqSpec("UCB", beta=0.2), w.candidates)
    assert float((qucb - ucb).abs().max()) < 5e-3


def test_minimisation_is_maximisation_of_negated_target():
    """Metamorphic property the reference tests (tests/integration/test_minimization.py:41-78)."""
    w = numeric_grid_workload(N=150, d=3, n=20, seed=8)
    om_max = oracle_model(w)
    w_neg = numeric_grid_workload(N=150, d=3, n=20, seed=8)
    w_neg.train_y = -w.train_y
    om_min = oracle_model(w_neg)
    mu_a, var_a = oracle.posterior(om_max, w.candidates)
    mu_b, var_b = oracle.posterior(om_min, w.candidates)
    assert torch.allclose(mu_a, -mu_b, atol=1e-12) and torch.allclose(var_a, var_b, atol=1e-12)
    z = oracle.sobol_normal_samples(512, 1, 1)[:, 0]
    for kind in ("qLogEI", "qEI", "EI", "UCB", "PM"):
        a = oracle.AcqSpec(kind)
        a.best_f = oracle.best_f_from_training(om_max, w.train_x, a)
        b = oracle.AcqSpec(kind, obj_scale=-1.0)
        b.best_f = oracle.best_f_from_training(om_min, w.train_x, b)
        va = oracle.acq_values(om_max, a, w.candidates, z)
        vb = oracle.acq_values(om_min, b, w.candidates, -z if kind.startswith("q") else None)
        assert torch.allclose(va, vb, rtol=1e-4, atol=1e-6), kind


def test_joint_scores_reduce_to_q1_and_match_brute_force():
    w = numeric_grid_workload(N=120, d=3, n=18, seed=9)
    om = oracle_model(w)
    acq = oracle.AcqSpec("qLogEI")
    acq.best_f = oracle.best_f_from_training(om, w.train_x, acq)
    z = oracle.sobol_normal_samples(256, 3, 5)
    pend = w.candidates[:2]
    cand = w.candidates[2:40]
    got = oracle.acq_values_joint(om, acq, cand, pend, z)
    # brute force with the full joint posterior of each [x*; pending] batch
    for i in (0, 7, 21):
        m, cov = oracle.posterior_joint(om, np.vstack([cand[i:i + 1], pend]))
        L = torch.linalg.cholesky(cov)
        y = m + z @ L.T
        li = oracle.reference_path._log_fatplus(y - acq.best_f, acq.tau_relu)
        val = torch.logsumexp(oracle.reference_path._fatmax(li, acq.tau_max), 0) - math.log(256)
        assert abs(float(val) - float(got[i])) < 1e-9
    none = oracle.acq_values_joint(om, acq, cand, np.zeros((0, 3)), z[:, :1])
    assert torch.allclose(none, oracle.acq_values(om, acq, cand, z[:, 0]))


def test_greedy_selection_semantics():
    w = numeric_grid_workload(N=90, d=3, n=15, seed=10)
    om = oracle_model(w)
    acq = oracle.AcqSpec("qLogEI")
    acq.best_f = oracle.best_f_from_training(om, w.train_x, acq)
    idx, vals = oracle.optimize_acqf_discrete(om, acq, w.candidates, q=4, sampler_seed=42, n_samples=128)
    assert len(set(idx)) == 4  # unique=True
    z1 = oracle.sobol_normal_samples(128, 1, 42)[:, 0]
    first = oracle.acq_values(om, acq, w.candidates, z1)
    assert idx[0] == int(torch.argmax(first)) and abs(vals[0] - float(first.max())) < 1e-12
    with pytest.raises(ValueError):
        oracle.optimize_acqf_discrete(om, oracle.AcqSpec("UCB"), w.candidates, q=2)
    # chunking never changes the numbers
    a = oracle.acq_values(om, acq, w.candidates, z1, chunk=7)
    assert torch.allclose(a, first, rtol=0, atol=1e-13)


def test_task_kernel_reduces_to_single_task_when_B_is_ones():
    w = task_workload(N_per_task=40, n_tasks=3, d_num=4, n_per_task=8, seed=1)
    w.task_covar = np.ones((3, 3))
    om = oracle_model(w)
    plain = oracle.KernelSpec("matern52", w.lengthscale[:4], [0, 1, 2, 3])
    om2 = oracle.build_model(plain, w.train_x[:, :4], w.train_y, w.bounds[:, :4], noise=w.noise[0])
    mu1, var1 = oracle.posterior(om, w.candidates)
    mu2, var2 = oracle.posterior(om2, w.candidates[:, :4])
    assert torch.allclose(mu1, mu2, atol=1e-10) and torch.allclose(var1, var2, atol=1e-10)


def test_sobol_base_samples_are_reproducible_standard_normal():
    z = oracle.sobol_normal_samples(512, 1, 1234)
    assert torch.equal(z, oracle.sobol_normal_samples(512, 1, 1234))
    assert abs(float(z.mean())) < 0.02 and abs(float(z.std()) - 1.0) < 0.02
    assert torch.isfinite(z).all()


@pytest.mark.parametrize("name", ["cfg1", "cfg2_slice", "task", "cfg4_slice"])
def test_golden_fixtures(name):
    """Committed fixtures (generated by tests/golden/make_golden.py from this oracle) pin the
    oracle against silent drift; they are not reference outputs (parity unpinned)."""
    data = json.loads((GOLDEN / f"{name}.json").read_text())
    from tests.golden.make_golden import WORKLOADS, evaluate

    fresh = evaluate(WORKLOADS[name]())
    for key, ref in data["values"].items():
        assert np.allclose(np.asarray(fresh[key]), np.asarray(ref), rtol=1e-9, atol=1e-12), key


# --------------------------------------------------------------------------------------
# Independent checks of the parts no second implementation covers (VERDICT r1, weak #1)
# --------------------------------------------------------------------------------------
def test_qlogei_matches_arbitrary_precision_definition():
    """qLogEI restated from its published definition in 60-digit arithmetic (mpmath), independent of the
    oracle's float64 branches (log-softplus tail switch at t < -30, logaddexp, logsumexp):
        fatplus(x; tau) = tau * ( log(1 + e^{x/tau}) + 0.1 / (1 + (x/tau)^2) ),   tau = 1e-6
        qLogEI          = log( (1/S) sum_s fatplus(o_s - best_f) )                (q = 1: fatmax is the identity)."""
    import mpmath as mp

    mp.mp.dps = 60
    z = oracle.sobol_normal_samples(128, 1, 77)[:, 0]
    cases = [(0.3, 0.04, 0.9), (1.2, 0.25, 1.0), (-0.5, 1e-4, 0.1), (2.0, 1e-10, 1.0), (0.999999, 1e-6, 1.0),
             (0.0, 9.0, 0.5), (5.0, 0.01, -3.0)]
    for mu, var, best in cases:
        for a in (1.0, -1.0):
            acq = oracle.AcqSpec("qLogEI", best_f=best, obj_scale=a)
            got = float(oracle.reference_path.acq_from_moments(acq, np.array([mu]), np.array([var]), z))
            tau = mp.mpf(10) ** -6
            tot = mp.mpf(0)
            for zs in z.tolist():
                x = (mp.mpf(a) * (mp.mpf(mu) + mp.sqrt(mp.mpf(var)) * mp.mpf(zs)) - mp.mpf(best)) / tau
                tot += tau * (mp.log1p(mp.e**x) + mp.mpf("0.1") / (1 + x * x))
            want = float(mp.log(tot / len(z)))
            assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), (mu, var, best, a, got, want)


def test_fatmax_matches_arbitrary_precision_definition():
    """fatmax(x; tau) = M + tau * log sum_i (1 + (M - x_i)/(alpha tau))^-alpha, alpha = 2 (q > 1 reduction of qLogEI)."""
    import mpmath as mp

    mp.mp.dps = 50
    g = torch.Generator().manual_seed(3)
    x = torch.randn(5, 4, generator=g, dtype=torch.float64) * 3.0 - 12.0
    got = oracle.reference_path._fatmax(x, 1e-2, dim=-1)
    for r in range(5):
        xs = [mp.mpf(v) for v in x[r].tolist()]
        M = max(xs)
        tau = mp.mpf("0.01")
        want = M + tau * mp.log(sum((1 + (M - v) / (2 * tau)) ** -2 for v in xs))
        assert abs(float(got[r]) - float(want)) < 1e-12


def test_qucb_centres_on_the_sample_mean():
    """botorch ``qUpperConfidenceBound._sample_forward``: ``mean = obj.mean(dim=0)`` (the MC sample mean) and
    ``mean + sqrt(beta*pi/2) * |obj - mean|``; with scrambled Sobol samples mean(z) != 0, so this differs from
    centring on the posterior mean.  Brute force over the samples, both orientations."""
    z = oracle.sobol_normal_samples(512, 1, 1234)[:, 0]
    assert abs(float(z.mean())) > 1e-6  # the distinction is observable
    mu, var = torch.tensor([0.7, -1.3], dtype=torch.float64), torch.tensor([0.09, 2.0], dtype=torch.float64)
    for a in (1.0, -1.0):
        acq = oracle.AcqSpec("qUCB", beta=0.2, obj_scale=a, obj_shift=0.25)
        got = oracle.reference_path.acq_from_moments(acq, mu, var, z)
        obj = a * (mu[None, :] + var.sqrt()[None, :] * z[:, None]) + 0.25  # (S, B)
        m = obj.mean(0)
        want = (m + math.sqrt(0.2 * math.pi / 2) * (obj - m).abs()).mean(0)
        assert torch.allclose(got, want, rtol=0, atol=1e-13)
        # closed form used by the CUDA kernels: mo + so*mean(z) + c*|so|*mean|z - mean z|
        mo, so = a * mu + 0.25, a * var.sqrt()
        closed = mo + so * z.mean() + math.sqrt(0.2 * math.pi / 2) * so.abs() * (z - z.mean()).abs().mean()
        assert torch.allclose(got, closed, rtol=0, atol=1e-12)


def test_sobol_normal_recipe_against_scipy():
    """The base-sample recipe (SURVEY A.6): torch SobolEngine(scramble=True, seed) uniforms ->
    v = 0.5 + (1 - eps)(u - 0.5) -> Phi^-1(v).  The uniforms come from the same torch engine botorch uses (its
    scrambling is torch's own, so no second library reproduces it bit for bit); checked here are (i) the
    unscrambled engine against scipy's Joe-Kuo Sobol points, (ii) the inverse-CDF transform against scipy's
    norm.ppf, (iii) the 2-D draw used for q = 2 rounds keeps column 0 a valid 1-D normal sample set."""
    from scipy.stats import qmc

    u_t = torch.quasirandom.SobolEngine(dimension=3, scramble=False).draw(64, dtype=torch.float64).numpy()
    u_s = qmc.Sobol(d=3, scramble=False, bits=30).random(64)
    assert np.allclose(np.sort(u_t, axis=0), np.sort(u_s, axis=0), atol=1e-9)
    eng = torch.quasirandom.SobolEngine(dimension=1, scramble=True, seed=1234)
    u = eng.draw(512, dtype=torch.float64)
    v = 0.5 + (1.0 - np.finfo(np.float64).eps) * (u.numpy() - 0.5)
    z = oracle.sobol_normal_samples(512, 1, 1234).numpy()
    assert np.allclose(z, norm.ppf(v), rtol=1e-11, atol=1e-12)
    assert 0.0 <= float(u.min()) and float(u.max()) < 1.0
    z2 = oracle.sobol_normal_samples(512, 2, 1234)
    assert z2.shape == (512, 2) and torch.isfinite(z2).all()


def test_standardize_and_noise_conventions():
    """botorch ``Standardize(m=1)``: unbiased std, std < 1e-8 -> 1; homoskedastic noise floored at 1e-4
    (MIN_INFERRED_NOISE_LEVEL, presets/baybe.py:129-144); posterior un-transform mu = ybar + s mu~, var = s^2 var~."""
    spec = oracle.KernelSpec("matern52", [0.5], [0])
    X = np.array([[0.1], [0.4], [0.8]])
    y = np.array([1.0, 3.0, 8.0])
    m = oracle.build_model(spec, X, y, np.array([[0.0], [1.0]]), noise=1e-3)
    assert abs(m.y_mean - 4.0) < 1e-15 and abs(m.y_std - float(np.std(y, ddof=1))) < 1e-15
    const = oracle.build_model(spec, X, np.array([2.0, 2.0, 2.0]), np.array([[0.0], [1.0]]), noise=1e-3)
    assert const.y_std == 1.0
    # explicit K^-1 formulas (no Cholesky) for the posterior in original units
    Xn = torch.tensor(X)
    K = oracle.kernel_matrix(spec, Xn, Xn) + 1e-3 * torch.eye(3, dtype=torch.float64)
    xs = np.array([[0.55]])
    ks = oracle.kernel_matrix(spec, torch.tensor(xs), Xn)
    yt = torch.tensor((y - 4.0) / np.std(y, ddof=1))
    Kinv = torch.linalg.inv(K)
    mu_ref = 4.0 + np.std(y, ddof=1) * float(ks @ Kinv @ yt)
    var_ref = np.var(y, ddof=1) * float(1.0 - ks @ Kinv @ ks.T)
    mu, var = oracle.posterior(m, xs)
    assert abs(float(mu) - mu_ref) < 1e-10 and abs(float(var) - var_ref) < 1e-10


def test_qnei_conditional_form_equals_the_joint_cholesky():
    """acq_values_qnei (conditional form: samples of [baseline; pending] once, the new point from its Cholesky row)
    against the definition evaluated candidate by candidate from the full joint posterior of
    [baseline; pending; x] (oracle.posterior_joint + Cholesky), same base samples."""
    from oracle import reference_path as rp

    w = numeric_grid_workload(N=60, d=4, n=12, seed=0)
    om = oracle_model(w)
    nb = 12
    for p, a in ((0, 1.0), (2, 1.0), (3, -1.0)):
        acq = oracle.AcqSpec("qEI", obj_scale=a, obj_shift=0.1)
        P = w.candidates[:p]
        z = oracle.sobol_normal_samples(128, nb + p + 1, 3)
        got = oracle.acq_values_qnei(om, acq, w.candidates[5:17], P, z)
        ref = []
        for x in w.candidates[5:17]:
            A = np.vstack([w.train_x, P, x[None]]) if p else np.vstack([w.train_x, x[None]])
            mu, cov = rp.posterior_joint(om, A)
            L = rp._chol_with_jitter(cov.unsqueeze(0))[0]
            o = a * (mu[None] + z @ L.T) + 0.1
            ref.append(float((o[:, nb:].amax(-1) - o[:, :nb].amax(-1)).clamp_min(0).mean()))
        assert np.abs(np.array(ref) - got.numpy()).max() < 1e-7
        assert float(got.max()) > 0


def test_leave_one_out_closed_form_equals_brute_force_refits():
    """The fit criterion of transfer-learning spaces (presets/baybe.py:270-281): the closed form used by the device
    kernel and its host twin -- sigma_i^2 = 1/[K^-1]_ii, mu_i = y_i - alpha_i sigma_i^2  [U: gpytorch
    LeaveOneOutPseudoLikelihood] -- against n explicit refits that leave one observation out and evaluate its
    Gaussian predictive log density (noisy observation)."""
    from tests.helpers import HostMLL

    rng = np.random.default_rng(7)
    n, d = 9, 3
    X = rng.random((n, d))
    y = np.sin(3 * X[:, 0]) + X[:, 1] ** 2 + 0.1 * rng.standard_normal(n)
    ls, noise, c = np.array([0.7, 0.9, 1.1]), 0.05, 0.2
    theta = np.concatenate([ls, [noise, c], [1.0]])
    got, _, ok = HostMLL(X, y, None, 1, "matern52", criterion="loo")(theta)
    assert ok

    def kern(A, B):
        r = np.sqrt((((A[:, None, :] - B[None, :, :]) / ls) ** 2).sum(-1))
        return (1 + np.sqrt(5) * r + 5 / 3 * r * r) * np.exp(-np.sqrt(5) * r)

    ref = 0.0
    for i in range(n):
        m = np.arange(n) != i
        Kmm = kern(X[m], X[m]) + noise * np.eye(n - 1)
        kim = kern(X[i : i + 1], X[m])[0]
        sol = np.linalg.solve(Kmm, np.stack([y[m] - c, kim], axis=1))
        mu = c + kim @ sol[:, 0]
        var = 1.0 + noise - kim @ sol[:, 1]
        ref += -0.5 * np.log(2 * np.pi * var) - 0.5 * (y[i] - mu) ** 2 / var
    assert abs(got - ref) < 1e-9 * max(1.0, abs(ref))


def test_fp32_distance_error_of_the_fused_shape_table_is_within_its_kernel_matrix_bound():
    """The kernel-matrix bound of tests/test_gpu_fused_shapes.py (kmat_tol) covers distances formed as the kernels form
    them, |a|^2 + |b|^2 - 2 a.b in fp32 on the kernels' centred, scaled rows: the error of that form alone, against
    the oracle, at every shape of the table."""
    from tests.test_gpu_fused_shapes import CASES, kernel_units, kmat_tol

    def k_of_t(family, t):
        if family == "rbf":
            return np.exp2(-t)
        r = np.sqrt(np.maximum(t, 0.0))
        return (1.0 + r) * np.exp(-r) if family == "matern32" else (1.0 + r + t / 3.0) * np.exp(-r)

    for name, case in CASES.items():
        w = case.make()
        if w.family == "matern12" or case.fused == "k_fused<3, true, 0, 0>":
            continue  # Matern-1/2: no GEMM-form kernel; wide rows: test_gpu_wide.py's bound
        a, b = (v.astype(np.float32) for v in kernel_units(w))
        t = ((a * a).sum(axis=1, dtype=np.float32)[:, None] + (b * b).sum(axis=1, dtype=np.float32)[None, :]
             - np.float32(2.0) * (a @ b.T))
        om = oracle_model(w)
        Kref = oracle.kernel_matrix(om.spec, (torch.from_numpy(w.candidates) - om.lo) / om.rng, om.Xn).numpy()
        K32 = k_of_t(w.family, t.astype(np.float64))
        if w.task_col is None:
            K32 = K32 * float(w.outputscale or 1.0)
        else:
            tc, tt = (x[:, w.task_col].astype(int) for x in (w.candidates, w.train_x))
            K32 = K32 * w.task_covar[tc][:, tt]
        err = float(np.abs(K32 - Kref).max())
        assert err <= kmat_tol(w, False) * max(1.0, float(np.abs(Kref).max())), (name, err)
