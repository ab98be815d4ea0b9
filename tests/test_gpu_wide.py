"""GPU parity tests of the wide-feature path (wide.cu: K-chunked wgmma distance GEMM + the
K*-reading posterior kernel) against the float64 CPU oracle: float layouts with d in the
hundreds, and bit-packed binary fingerprints at the BASELINE config-4 shape (d = 2048 bits,
n = 512, ScaleKernel(RBF)) at a candidate count the oracle finishes in seconds.

Tolerances are those of tests/test_gpu_parity.py (same fp32 engine, same oracle), except the
kernel matrix: the GEMM-form distance t = |a|^2 + |b|^2 - 2 a.b is formed in fp32 from norms that
grow with d, so |dK| <= 2e-6 * max(1, d/32) here (fp32 rounding of O(d)-sized norms; the
posterior tolerances are unchanged).
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import AcqConfig, DeviceGP, sobol_normal_samples
from baybe_b200.engine import decode_best
from baybe_b200.synthetic import fingerprint_workload, numeric_grid_workload, pack_bits, task_workload
from tests.helpers import oracle_model, score_bounds

pytestmark = pytest.mark.gpu


def _gp(w, dev):
    return DeviceGP(device=dev, **w.gp_kwargs())


def _var_tol(om):
    return 2e-5 * float(om.spec.outputscale or 1.0) * om.y_std**2


WIDE = {
    # n_pad * d_pad * 4 > 56 KB  ->  wide model
    "d100_n200_m52": lambda: numeric_grid_workload(N=3000, d=100, n=200, seed=11,
                                                   lengthscale=np.linspace(1.5, 4.0, 100)),
    "d333_n130_rbf_scaled": lambda: numeric_grid_workload(N=1100, d=333, n=130, family="rbf", seed=12,
                                                          outputscale=1.7, lengthscale=6.0),
    "d40_n512_m32": lambda: numeric_grid_workload(N=2500, d=40, n=512, family="matern32", seed=13,
                                                  lengthscale=2.0),
    # n > 512: always wide, several V column panels per tile
    "d12_n700_m52": lambda: numeric_grid_workload(N=2000, d=12, n=700, seed=14, lengthscale=1.2),
    "d40_n1024_rbf": lambda: numeric_grid_workload(N=1800, d=40, n=1024, family="rbf", seed=15, lengthscale=2.5,
                                                   outputscale=0.8),
    "fp2048_n512": lambda: fingerprint_workload(N=2300, d=2048, n=512, seed=1),
    "fp1000_n300": lambda: fingerprint_workload(N=1500, d=1000, n=300, seed=2, density=0.1, family="matern52",
                                                ls_factor=0.25, outputscale=None),
}


def _inputs(w, dev, name):
    """Device candidate matrix in the layout the workload is meant for."""
    if name.startswith("fp"):
        return torch.from_numpy(pack_bits(w.candidates)).to(dev)
    return torch.from_numpy(w.candidates).to(dev, torch.float32)


@pytest.mark.parametrize("name", list(WIDE))
def test_wide_model_flag_and_kernel_matrix(name, cuda_device):
    w = WIDE[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    assert gp.model.wide == 1
    K = gp.kernel_matrix(_inputs(w, cuda_device, name)).double().cpu()
    Xn = (torch.from_numpy(w.candidates) - om.lo) / om.rng
    Kref = oracle.kernel_matrix(om.spec, Xn, om.Xn)
    assert K.shape == Kref.shape
    d = w.candidates.shape[1]
    assert float((K - Kref).abs().max()) <= 2e-6 * max(1.0, d / 32) * max(1.0, float(Kref.abs().max()))


@pytest.mark.parametrize("name", list(WIDE))
def test_wide_posterior(name, cuda_device):
    w = WIDE[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    mu, var = gp.posterior(_inputs(w, cuda_device, name))
    mu, var = mu.double().cpu(), var.double().cpu()
    mu_ref, var_ref = oracle.posterior(om, w.candidates)
    assert float((mu - mu_ref).abs().max()) <= 5e-5 * max(1.0, float(mu_ref.abs().max()))
    assert float((var - var_ref).abs().max()) <= _var_tol(om)
    assert float(var.min()) > 0


@pytest.mark.parametrize("kind", ["qLogEI", "qEI", "UCB", "LogEI"])
@pytest.mark.parametrize("name", ["d100_n200_m52", "fp2048_n512", "d12_n700_m52"])
def test_wide_scores_and_argmax(kind, name, cuda_device):
    w = WIDE[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    oacq = oracle.AcqSpec(kind=kind)
    oacq.best_f = oracle.best_f_from_training(om, w.train_x, oacq)
    acq = AcqConfig(kind=kind, best_f=oacq.best_f)
    z = sobol_normal_samples(512, 1, seed=1234)
    scores, key = gp.score(acq, _inputs(w, cuda_device, name), z[:, 0] if acq.is_mc else None)
    ref, bound = score_bounds(om, oacq, w.candidates, z[:, 0] if oacq.is_mc else None)  # hard per-row bound
    got = scores.double().cpu()
    err = (got - ref).abs()
    worst = int(torch.argmax(err - bound))
    assert bool((err <= bound).all()), f"{kind}: row {worst} |err| {float(err[worst]):.3e} > bound {float(bound[worst]):.3e}"
    val, idx = decode_best(key)
    assert idx == int(torch.argmax(scores).item()) and val == float(scores[idx].item())
    ref_idx = int(torch.argmax(ref))
    assert float(ref[idx]) >= float(ref[ref_idx]) - float(bound[ref_idx] + bound[idx])


@pytest.mark.parametrize("P", [1, 5])
@pytest.mark.parametrize("name", ["d100_n200_m52", "fp2048_n512", "fp1000_n300", "d40_n1024_rbf"])
def test_wide_joint_scores_with_pending_points(name, P, cuda_device):
    """Sequential-greedy round on the wide path: pending rows become 64 extra K columns of k_kmat_tc and the
    cross-covariances are contracted from the K* block in the workspace."""
    w = WIDE[name]()
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    oacq = oracle.AcqSpec(kind="qLogEI")
    oacq.best_f = oracle.best_f_from_training(om, w.train_x, oacq)
    acq = AcqConfig(kind="qLogEI", best_f=oacq.best_f)
    rng = np.random.default_rng(P)
    pend_rows = rng.choice(len(w.candidates), size=P, replace=False)
    pending = w.candidates[pend_rows]
    keep = np.setdiff1d(np.arange(len(w.candidates)), pend_rows)[:900]
    cand = w.candidates[keep]
    z = sobol_normal_samples(512, 1 + P, seed=99)
    x = torch.from_numpy(pack_bits(cand)).to(cuda_device) if name.startswith("fp") else \
        torch.from_numpy(cand).to(cuda_device, torch.float32)
    got = gp.score_joint(acq, x, pending, z).double().cpu()
    ref = oracle.acq_values_joint(om, oacq, cand, pending, z)
    _, bound = score_bounds(om, oacq, cand, z[:, 0])
    bound = 2.0 * bound + 2e-3  # candidate row's own bound, doubled for the cross-covariance terms; every row
    err = (got - ref).abs()
    worst = int(torch.argmax(err - bound))
    assert bool((err <= bound).all()), (name, P, worst, float(err[worst]), float(bound[worst]))
    win = int(torch.argmax(got))
    assert float(ref[win]) >= float(ref.max()) - float(bound[win] + bound[int(torch.argmax(ref))])


@pytest.mark.parametrize("S", [128, 512])
def test_wide_tabulated_qlogei_matches_exact_sample_loop(S, cuda_device):
    """K*-reading kernel: the qLogEI table is built once per call (k_mc_table) and shared by all blocks."""
    w = numeric_grid_workload(N=50_000, d=72, n=200, seed=23, lengthscale=2.5)
    gp = _gp(w, cuda_device)
    x = torch.from_numpy(w.candidates).to(cuda_device, torch.float32)
    z = sobol_normal_samples(S, 1, seed=5)[:, 0]
    acq = AcqConfig(kind="qLogEI", best_f=gp.best_f(AcqConfig(kind="qLogEI")))
    scores, _ = gp.score(acq, x, z)
    mu, var = gp.posterior(x)
    exact = torch.ops.baybe_b200.acq_score(mu, var, z.to(cuda_device, torch.float32), 0, acq.params())
    assert torch.allclose(scores, exact, rtol=2e-4, atol=2e-4), float((scores - exact).abs().max())


def test_bits_and_float_layouts_agree(cuda_device):
    """The bit-linear form and the generic float form are two roundings of the same distances."""
    w = WIDE["fp2048_n512"]()
    gp = _gp(w, cuda_device)
    om = oracle_model(w)
    mu_b, var_b = gp.posterior(torch.from_numpy(pack_bits(w.candidates)).to(cuda_device))
    mu_f, var_f = gp.posterior(torch.from_numpy(w.candidates).to(cuda_device, torch.float32))
    mu_d, var_d = gp.posterior(torch.from_numpy(w.candidates).to(cuda_device).t().contiguous().t())  # col-major f64
    assert torch.equal(mu_f, mu_d) and torch.equal(var_f, var_d)
    assert float((mu_b - mu_f).abs().max()) <= 2e-5 * max(1.0, float(mu_f.abs().max()))
    assert float((var_b - var_f).abs().max()) <= 2 * _var_tol(om)  # each is within _var_tol of the oracle


def test_wide_blocks_and_offsets(cuda_device):
    """More candidates than one K* workspace block (33,792 rows at n = 256): block seams, index offsets, keep mask."""
    w = numeric_grid_workload(N=80_000, d=72, n=256, seed=21, lengthscale=2.5)
    gp = _gp(w, cuda_device)
    assert gp.model.wide == 1 and gp.model.wide_ws_rows < 80_000
    x = torch.from_numpy(w.candidates).to(cuda_device, torch.float32)
    z = sobol_normal_samples(512, 1, seed=3)
    acq = AcqConfig(kind="qLogEI", best_f=gp.best_f(AcqConfig(kind="qLogEI")))
    scores, key = gp.score(acq, x, z[:, 0])
    _, idx = decode_best(key)
    assert idx == int(torch.argmax(scores).item())
    # any sub-range scored on its own gives the same numbers (no dependence on the block position)
    lo, hi = 33_000, 35_500
    sub, key_sub = gp.score(acq, x[lo:hi], z[:, 0], index_offset=lo)
    assert torch.equal(sub, scores[lo:hi])
    assert decode_best(key_sub)[1] == lo + int(torch.argmax(sub).item())
    keep = torch.ones(x.shape[0], dtype=torch.uint8, device=cuda_device)
    keep[idx] = 0
    masked = scores.clone()
    masked[idx] = -float("inf")
    _, key2 = gp.score(acq, x, z[:, 0], keep=keep, want_scores=False)
    assert decode_best(key2)[1] == int(torch.argmax(masked).item())
    om = oracle_model(w)
    mu_ref, var_ref = oracle.posterior(om, w.candidates[37_800:38_000])
    mu, var = gp.posterior(x)
    assert float((mu[37_800:38_000].double().cpu() - mu_ref).abs().max()) <= 5e-5 * max(1.0, float(mu_ref.abs().max()))
    assert float((var[37_800:38_000].double().cpu() - var_ref).abs().max()) <= _var_tol(om)


def test_wide_task_model(cuda_device):
    """Task column + wide numeric part: the task covariance is applied in the K* epilogue."""
    w = task_workload(N_per_task=500, n_tasks=3, d_num=90, n_per_task=60, seed=5)
    om = oracle_model(w)
    gp = _gp(w, cuda_device)
    assert gp.model.wide == 1
    mu, var = gp.posterior(torch.from_numpy(w.candidates).to(cuda_device, torch.float32))
    mu_ref, var_ref = oracle.posterior(om, w.candidates)
    prior = float(np.max(np.diag(w.task_covar))) * float(w.outputscale or 1.0)
    assert float((mu.double().cpu() - mu_ref).abs().max()) <= 5e-5 * max(1.0, float(mu_ref.abs().max()))
    assert float((var.double().cpu() - var_ref).abs().max()) <= 2e-5 * prior * om.y_std**2


def test_wide_errors_are_loud(cuda_device):
    w = numeric_grid_workload(N=500, d=20, n=64)  # not wide
    gp = _gp(w, cuda_device)
    assert gp.model.wide == 0
    with pytest.raises(NotImplementedError):
        gp.posterior(torch.zeros(10, 3, dtype=torch.uint8))  # bit-packed rows need a wide model
    wm = numeric_grid_workload(N=300, d=100, n=200, family="matern12", seed=1)
    gm = _gp(wm, cuda_device)
    with pytest.raises(NotImplementedError):
        gm.posterior(torch.from_numpy(wm.candidates))  # Matern-1/2 is not offered on the GEMM-form wide path
    fp = WIDE["fp1000_n300"]()
    gf = _gp(fp, cuda_device)
    with pytest.raises(ValueError):
        gf.posterior(torch.zeros(10, 100, dtype=torch.uint8))  # wrong packed width (needs 125 bytes)
