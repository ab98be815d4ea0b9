"""GPU parity tests: the CUDA path (through torch custom ops -> C ABI) against the float64 CPU
oracle on identical seeded inputs.

Stated tolerances (float32 engine vs float64 oracle, standardised-target units ~ O(1)):
  kernel matrix   |dK|        <= 3e-6
  posterior mean  |dmu|       <= 5e-5 * max(1, |mu|_inf)   (fp32 dot product against alpha)
  posterior var   |dvar|      <= 2e-5 * prior variance     (fp16x3 tensor-core contraction)
  acquisition     rtol 1e-4 / atol 0.1 is what the reference itself accepts
                  (/root/reference/tests/integration/test_minimization.py:78); we hold, for EVERY row,
                  |d score| <= 2e-4 + 1e-4*|score| + 1.5 * (score change the posterior tolerance above can
                  cause at that row, evaluated by the oracle) -- tests/helpers.py::score_bounds.
  recommended index: identical to the oracle whenever no other row's score interval overlaps the
                  oracle winner's; otherwise the GPU winner's oracle score lies within the two bounds.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import AcqConfig, DeviceGP, sobol_normal_samples
from baybe_b200.engine import decode_best
from baybe_b200.synthetic import (mixed_small_workload, numeric_grid_workload, task_workload)
from tests.helpers import oracle_model, score_bounds

pytestmark = pytest.mark.gpu


def _gp(w, dev):
    return DeviceGP(device=dev, **w.gp_kwargs())


def _var_tol(om):
    prior = float(om.spec.outputscale or 1.0)
    if om.spec.task_covar is not None:
        prior *= float(np.max(np.diag(om.spec.task_covar)))
    return 2e-5 * prior * om.y_std**2


WORKLOADS = {
    "cfg2_small": lambda: numeric_grid_workload(N=6000, d=20, n=256),
    "cfg1": mixed_small_workload,
    "n100_d7_rbf_scaled": lambda: numeric_grid_workload(N=1500, d=7, n=100, family="rbf", outputscale=2.5,
                                                        lengthscale=np.linspace(0.4, 1.5, 7), seed=3),
    "n300_d12_m32": lambda: numeric_grid_workload(N=2000, d=12, n=300, family="matern32", seed=4,
                                                  lengthscale=0.8),
    "n512_d20_m52": lambda: numeric_grid_workload(N=3000, d=20, n=512, seed=5),
    # 30 < d <= 62 with n_pad <= 256: the K = 64 augmented distance GEMM
    "n200_d48_m52": lambda: numeric_grid_workload(N=2000, d=48, n=200, seed=7, lengthscale=2.0),
    "n33_d3_m12": lambda: numeric_grid_workload(N=700, d=3, n=33, family="matern12", seed=6,
                                                lengthscale=0.5, levels=9),
    "task4": lambda: task_workload(N_per_task=800, n_tasks=4, d_num=6, n_per_task=40, seed=2),
}


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_kernel_matrix(name, cuda_device):
    w = WORKLOADS[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    K = gp.kernel_matrix(torch.from_numpy(w.candidates)).double().cpu()
    Xn = (torch.from_numpy(w.candidates) - om.lo) / om.rng
    Kref = oracle.kernel_matrix(om.spec, Xn, om.Xn)
    scale = float(Kref.abs().max())
    assert K.shape == Kref.shape
    # GEMM-form distances (gpytorch's Distance._sq_dist, here with |a|^2 + |b|^2 inside the tensor-core GEMM) are
    # accumulated in float32: |dt| ~ 2^-22 (|a|^2 + |b|^2), |dk/dt| <= 1/6 -> 3e-6 covers scaled norms up to ~40
    assert float((K - Kref).abs().max()) <= 3e-6 * max(1.0, scale)


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_posterior_tensor_core_path(name, cuda_device):
    w = WORKLOADS[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    mu, var = gp.posterior(torch.from_numpy(w.candidates))
    mu, var = mu.double().cpu(), var.double().cpu()
    mu_ref, var_ref = oracle.posterior(om, w.candidates)
    assert float((mu - mu_ref).abs().max()) <= 5e-5 * max(1.0, float(mu_ref.abs().max()))
    assert float((var - var_ref).abs().max()) <= _var_tol(om)
    assert float(var.min()) > 0


@pytest.mark.parametrize("name", ["cfg2_small", "task4", "n100_d7_rbf_scaled"])
def test_posterior_simt_diagnostic_path(name, cuda_device):
    w = WORKLOADS[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    mu, var = gp.posterior_simt(torch.from_numpy(w.candidates))
    mu_ref, var_ref = oracle.posterior(om, w.candidates)
    assert float((mu.double().cpu() - mu_ref).abs().max()) <= 5e-5 * max(1.0, float(mu_ref.abs().max()))
    assert float((var.double().cpu() - var_ref).abs().max()) <= _var_tol(om)


def test_posterior_at_training_points_is_small_and_positive(cuda_device):
    w = WORKLOADS["cfg2_small"]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    mu, var = gp.posterior(torch.from_numpy(w.train_x))
    _, var_ref = oracle.posterior(om, w.train_x)
    rel = ((var.double().cpu() - var_ref).abs() / var_ref).max()
    assert float(rel) < 5e-3  # cancellation site: var ~ noise level, abs error ~1e-6
    assert float(var.min()) > 0


@pytest.mark.parametrize("layout", ["row_f32", "col_f32", "row_f64", "col_f64", "row_f32_padded"])
def test_candidate_layouts_agree(layout, cuda_device):
    w = WORKLOADS["cfg2_small"]()
    gp = _gp(w, cuda_device)
    base = torch.from_numpy(w.candidates)
    ref_mu, ref_var = gp.posterior(base.to(cuda_device, torch.float32))
    if layout == "row_f32":
        x = base.to(cuda_device, torch.float32)
    elif layout == "col_f32":
        x = base.to(cuda_device, torch.float32).t().contiguous().t()
    elif layout == "row_f64":
        x = base.to(cuda_device)
    elif layout == "col_f64":  # what the reference's to_tensor produces (utils/dataframe.py:68-81)
        x = base.to(cuda_device).t().contiguous().t()
    else:
        buf = torch.zeros(base.shape[0], 24, device=cuda_device, dtype=torch.float32)
        buf[:, :20] = base.to(cuda_device, torch.float32)
        x = buf[:, :20]
    assert x.shape == base.shape
    mu, var = gp.posterior(x)
    # all layouts are converted to the same fp32 values on load: bit-identical results
    assert torch.equal(mu, ref_mu) and torch.equal(var, ref_var)


MC = ["qLogEI", "qEI", "qUCB", "qSR", "qPI"]
ANALYTIC = ["UCB", "EI", "LogEI", "PI", "PM", "PSTD"]


def _score_tols(kind):
    if kind in ("qLogEI", "LogEI"):
        return 5e-3, 2e-3  # log scale: atol, rtol
    return 2e-4, 2e-3


@pytest.mark.parametrize("kind", MC + ANALYTIC)
@pytest.mark.parametrize("name,minimize", [("cfg2_small", False), ("cfg1", True), ("task4", False)])
def test_fused_scores_and_argmax(kind, name, minimize, cuda_device):
    w = WORKLOADS[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    a = -1.0 if minimize else 1.0
    oacq = oracle.AcqSpec(kind=kind, obj_scale=a)
    oacq.best_f = oracle.best_f_from_training(om, w.train_x, oacq)
    z = sobol_normal_samples(512, 1, seed=1234)
    acq = AcqConfig(kind=kind, obj_scale=a, best_f=0.0)
    acq = AcqConfig(kind=kind, obj_scale=a, best_f=gp.best_f(acq))
    assert abs(acq.best_f - oacq.best_f) <= 5e-5 * max(1.0, abs(oacq.best_f))
    x = torch.from_numpy(w.candidates).to(cuda_device, torch.float32)
    scores, key = gp.score(acq, x, z[:, 0] if acq.is_mc else None)
    # hard per-row bound: float32 acquisition arithmetic + what the stated posterior tolerance can move the score
    ref, bound = score_bounds(om, oacq, w.candidates, z[:, 0] if oacq.is_mc else None)
    got = scores.double().cpu()
    err = (got - ref).abs()
    worst = int(torch.argmax(err - bound))
    assert bool((err <= bound).all()), (f"{kind}: row {worst} |err| {float(err[worst]):.3e} > bound "
                                        f"{float(bound[worst]):.3e} (ref {float(ref[worst]):.5f})")
    val, idx = decode_best(key)
    assert idx == int(torch.argmax(scores).item())  # first maximum, like torch.argmax
    assert val == float(scores[idx].item())
    # winner parity: identical to the oracle's winner unless the oracle's runner-up is within the winner's own bound
    ref_idx = int(torch.argmax(ref).item())
    ref_best = float(ref[ref_idx])
    assert float(ref[idx]) >= ref_best - float(bound[ref_idx] + bound[idx])
    contenders = torch.nonzero(ref + bound >= ref_best - float(bound[ref_idx])).reshape(-1)
    if contenders.numel() == 1:
        assert idx == ref_idx


def test_fused_matches_two_step_path_and_keep_mask(cuda_device):
    w = WORKLOADS["cfg2_small"]()
    gp = _gp(w, cuda_device)
    z = sobol_normal_samples(512, 1, seed=7)
    acq = AcqConfig(kind="qLogEI", best_f=gp.best_f(AcqConfig(kind="qLogEI")))
    x = torch.from_numpy(w.candidates).to(cuda_device, torch.float32)
    scores, key = gp.score(acq, x, z[:, 0])
    mu, var = gp.posterior(x)
    two_step = torch.ops.baybe_b200.acq_score(mu, var, z[:, 0].to(cuda_device, torch.float32),
                                              0, acq.params())
    assert torch.allclose(scores, two_step, rtol=1e-4, atol=1e-4)
    # exclude the winner: the next call must return the runner-up
    _, idx = decode_best(key)
    keep = torch.ones(x.shape[0], dtype=torch.uint8, device=cuda_device)
    keep[idx] = 0
    _, key2 = gp.score(acq, x, z[:, 0], keep=keep, want_scores=False)
    _, idx2 = decode_best(key2)
    masked = scores.clone()
    masked[idx] = -float("inf")
    assert idx2 == int(torch.argmax(masked).item())
    # shard offsets land in the decoded index
    _, key3 = gp.score(acq, x, z[:, 0], index_offset=1_000_000, want_scores=False)
    assert decode_best(key3)[1] == idx + 1_000_000


@pytest.mark.parametrize("minimize", [False, True])
@pytest.mark.parametrize("S", [64, 128, 256, 512])
def test_tabulated_qlogei_matches_exact_sample_loop(S, minimize, cuda_device):
    """The fused kernels evaluate qLogEI through the shared-table form (16 exact terms + tabulated fat tail, exact
    fallback rows); bb_acq_score sums every sample.  Both see the same (mu, var) and base samples."""
    w = WORKLOADS["cfg2_small"]()
    gp = _gp(w, cuda_device)
    a = -1.0 if minimize else 1.0
    z = sobol_normal_samples(S, 1, seed=11)[:, 0]
    acq = AcqConfig(kind="qLogEI", obj_scale=a, best_f=0.0)
    acq = AcqConfig(kind="qLogEI", obj_scale=a, best_f=gp.best_f(acq))
    x = torch.from_numpy(w.candidates).to(cuda_device, torch.float32)
    scores, key = gp.score(acq, x, z)
    mu, var = gp.posterior(x)
    exact = torch.ops.baybe_b200.acq_score(mu, var, z.to(cuda_device, torch.float32), 0, acq.params())
    assert torch.allclose(scores, exact, rtol=2e-4, atol=2e-4), float((scores - exact).abs().max())
    assert decode_best(key)[1] == int(torch.argmax(scores).item())
    # a much better incumbent pushes every row into the tabulated regime, a much worse one into the exact rows
    for shift in (-3.0, 3.0):
        acq2 = AcqConfig(kind="qLogEI", obj_scale=a, best_f=acq.best_f + shift)
        s2, _ = gp.score(acq2, x, z)
        e2 = torch.ops.baybe_b200.acq_score(mu, var, z.to(cuda_device, torch.float32), 0, acq2.params())
        assert torch.allclose(s2, e2, rtol=2e-4, atol=2e-4), (shift, float((s2 - e2).abs().max()))


def test_topk_and_argmax_ops(cuda_device):
    g = torch.Generator().manual_seed(0)
    s = torch.randn(100_000, generator=g).to(cuda_device)
    s[12345] = s[777] = s.max() + 1.0  # tie -> lowest index first
    vals, idx = torch.ops.baybe_b200.topk(s, None, 5)
    ref_vals, _ = torch.topk(s, 5)
    assert torch.equal(vals, ref_vals)
    assert idx[0].item() == 777 and idx[1].item() == 12345
    key = torch.ops.baybe_b200.argmax(s, None, 0)
    assert decode_best(key) == (float(s[777]), 777)
    keep = torch.ones_like(s, dtype=torch.uint8)
    keep[777] = 0
    assert decode_best(torch.ops.baybe_b200.argmax(s, keep, 0))[1] == 12345
    s_nan = s.clone()
    s_nan[5] = float("nan")
    assert decode_best(torch.ops.baybe_b200.argmax(s_nan, None, 0))[1] == 777
    empty = torch.zeros_like(keep)
    assert decode_best(torch.ops.baybe_b200.argmax(s, empty, 0))[1] == -1


@pytest.mark.parametrize("kind", ["qLogEI", "qEI", "qUCB", "qSR"])
@pytest.mark.parametrize("P", [1, 3, 7])
def test_joint_scores_with_pending_points(kind, P, cuda_device):
    w = WORKLOADS["cfg2_small"]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    oacq = oracle.AcqSpec(kind=kind)
    oacq.best_f = oracle.best_f_from_training(om, w.train_x, oacq)
    acq = AcqConfig(kind=kind, best_f=oacq.best_f)
    rng = np.random.default_rng(P)
    pend_rows = rng.choice(len(w.candidates), size=P, replace=False)
    pending = w.candidates[pend_rows]
    cand = np.delete(w.candidates, pend_rows, axis=0)[:1500]
    z = sobol_normal_samples(512, 1 + P, seed=99)
    got = gp.score_joint(acq, torch.from_numpy(cand), pending, z).double().cpu()
    ref = oracle.acq_values_joint(om, oacq, cand, pending, z)
    # joint scores see the candidate's moments AND its covariance with the pending points; the q=1 bound of the
    # candidate's own row, doubled for the cross terms, holds for every row (no outlier allowance)
    _, bound = score_bounds(om, oacq, cand, z[:, 0])
    bound = 2.0 * bound + 2e-3
    err = (got - ref).abs()
    worst = int(torch.argmax(err - bound))
    assert bool((err <= bound).all()), (kind, P, worst, float(err[worst]), float(bound[worst]))
    win = int(torch.argmax(got))
    assert float(ref[win]) >= float(ref.max()) - float(bound[win] + bound[int(torch.argmax(ref))])


def test_errors_are_loud(cuda_device):
    w = WORKLOADS["cfg1"]()
    gp = _gp(w, cuda_device)
    with pytest.raises(ValueError):
        gp.posterior(torch.zeros(10, 4))  # wrong column count
    with pytest.raises(ValueError):
        gp.score(AcqConfig(kind="qLogEI"), torch.from_numpy(w.candidates), None)  # no base samples
    big = numeric_grid_workload(N=1100, d=4, n=1100)
    with pytest.raises(NotImplementedError):
        DeviceGP(device=cuda_device, **big.gp_kwargs())  # n > BB_MAX_TRAIN
    with pytest.raises(ValueError):
        AcqConfig(kind="qKG")


def test_empty_and_tiny_candidate_sets(cuda_device):
    w = WORKLOADS["cfg1"]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    mu, var = gp.posterior(torch.zeros(0, 5))
    assert mu.numel() == 0 and var.numel() == 0
    one = w.candidates[:1]
    mu, var = gp.posterior(torch.from_numpy(one))
    mu_ref, var_ref = oracle.posterior(om, one)
    assert abs(float(mu) - float(mu_ref)) < 5e-4 * max(1, abs(float(mu_ref)))
    # ragged: N not a multiple of the 128-row tile
    for N in (127, 129, 191):
        mu, _ = gp.posterior(torch.from_numpy(w.candidates[:N]))
        assert mu.shape == (N,) and torch.isfinite(mu).all()
