"""Shapes of the fused scoring kernel that the other workloads leave out: a model whose V panel is only partly
filled (n_pad = 192 on the tensor-core path: three K* chunks in a four-sub-block panel), a ragged last tile, fewer
tiles than SMs (some warpgroup pairs take a single tile, most CTAs none), the gated single-launch pass at
n_pad = 192, and a small training set with many features, whose launch has room for only a few L^-1 stages.
Checked against the float64 oracle with the tolerances of test_gpu_parity.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import AcqConfig, DeviceGP, sobol_normal_samples
from baybe_b200.engine import decode_best
from baybe_b200.synthetic import numeric_grid_workload
from tests.helpers import oracle_model, score_bounds

pytestmark = pytest.mark.gpu


def _var_tol(om):
    prior = float(om.spec.outputscale or 1.0)
    return 2e-5 * prior * om.y_std**2


def _check_posterior_and_scores(w, dev, kinds=("qLogEI", "qEI", "UCB")):
    om = oracle_model(w)
    gp = DeviceGP(device=dev, **w.gp_kwargs())
    x = torch.from_numpy(w.candidates).to(dev, torch.float32)
    mu, var = gp.posterior(x)
    mu_ref, var_ref = oracle.posterior(om, w.candidates)
    assert float((mu.double().cpu() - mu_ref).abs().max()) <= 5e-5 * max(1.0, float(mu_ref.abs().max()))
    assert float((var.double().cpu() - var_ref).abs().max()) <= _var_tol(om)
    assert float(var.min()) > 0
    z = sobol_normal_samples(512, 1, seed=1234)
    for kind in kinds:
        oacq = oracle.AcqSpec(kind=kind, obj_scale=1.0)
        oacq.best_f = oracle.best_f_from_training(om, w.train_x, oacq)
        acq = AcqConfig(kind=kind, best_f=gp.best_f(AcqConfig(kind=kind)))
        scores, key = gp.score(acq, x, z[:, 0] if acq.is_mc else None)
        ref, bound = score_bounds(om, oacq, w.candidates, z[:, 0] if oacq.is_mc else None)
        err = (scores.double().cpu() - ref).abs()
        worst = int(torch.argmax(err - bound))
        assert bool((err <= bound).all()), f"{kind}: row {worst} |err| {float(err[worst]):.3e} > {float(bound[worst]):.3e}"
        val, idx = decode_best(key)
        assert idx == int(torch.argmax(scores).item())
        assert val == float(scores[idx].item())
        ref_idx = int(torch.argmax(ref).item())
        assert float(ref[idx]) >= float(ref[ref_idx]) - float(bound[ref_idx] + bound[idx])


@pytest.mark.parametrize("N", [4099, 1000, 129])
def test_partial_panel_n192_on_tensor_cores(N, cuda_device):
    """n = 150 -> n_pad = 192, d = 10: distances on the tensor cores (K = 32), three chunks, sub-block 3 of the
    panel unused.  N = 4099 ends in a ragged tile of 3 rows, 1000 gives 8 tiles (fewer than the SMs), 129 gives a
    full tile and a one-row tile."""
    w = numeric_grid_workload(N=N, d=10, n=150, seed=11, lengthscale=0.7)
    gp = DeviceGP(device=cuda_device, **w.gp_kwargs())
    assert gp.model.n_pad == 192 and gp.model.dist_k == 32
    _check_posterior_and_scores(w, cuda_device)


def test_ragged_tile_on_the_full_panel(cuda_device):
    """n = 256 (one full panel of four sub-blocks), a ragged last tile and fewer tiles than SMs."""
    w = numeric_grid_workload(N=5 * 128 + 77, d=20, n=256, seed=12)
    _check_posterior_and_scores(w, cuda_device, kinds=("qLogEI", "PI"))


def test_gated_pass_at_n192_is_bit_identical_to_resident(cuda_device):
    """The single-launch gated pass (rows published by the copy stream while the kernel runs; each consumer
    warpgroup waits for its tile's rows on its own) scores exactly as the resident pass at n_pad = 192."""
    w = numeric_grid_workload(N=300_001, d=10, n=150, seed=13, lengthscale=0.7)
    gp = DeviceGP(device=cuda_device, **w.gp_kwargs())
    assert gp.model.n_pad == 192
    z = sobol_normal_samples(512, 1, seed=5)
    acq = AcqConfig(kind="qLogEI", best_f=gp.best_f(AcqConfig(kind="qLogEI")))
    x_host = torch.from_numpy(w.candidates).to(torch.float32).pin_memory()
    keep = torch.ones(len(x_host), dtype=torch.uint8, device=cuda_device)
    keep[::9] = 0
    old = DeviceGP.OVERLAPPED_HOST_PASS
    try:
        DeviceGP.OVERLAPPED_HOST_PASS = True
        s_res, k_res = gp.score(acq, x_host.to(cuda_device), z[:, 0], keep=keep, index_offset=17)
        s_str, k_str = gp.score(acq, x_host, z[:, 0], keep=keep, index_offset=17)
    finally:
        DeviceGP.OVERLAPPED_HOST_PASS = old
    # the single gated launch ran (a shape outside its envelope would fall back to the block-wise pass)
    assert getattr(gp, "_gated_pass_pending", False)
    assert torch.equal(s_res, s_str) and int(k_res.item()) == int(k_str.item())
    gp.check_host_pass()
    assert np.isfinite(s_res.cpu().numpy()).all()


def test_few_training_points_many_features(cuda_device):
    """n = 50, d = 100: CUDA-core distances (d > 62) at n_pad = 64 with 100 features staged per candidate row.  Shared
    memory leaves room for 3 L^-1 stages; one chunk needs one tile in flight, so the model scores."""
    w = numeric_grid_workload(N=3000, d=100, n=50, seed=14, lengthscale=3.0)
    gp = DeviceGP(device=cuda_device, **w.gp_kwargs())
    assert gp.model.n_pad == 64 and not gp.model.wide
    _check_posterior_and_scores(w, cuda_device, kinds=("qLogEI", "EI"))
