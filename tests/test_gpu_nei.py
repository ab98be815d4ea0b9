"""qNEI / qLogNEI on the device: bb_joint_posterior against a float64 restatement, bb_nei_score row by row against the
float64 definition of tests/nei_oracle.py fed with the same moments, conditioning and base samples, greedy batches,
the 1M-row recommendation and real Campaign runs."""
from __future__ import annotations

import dataclasses
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import DeviceGP, noisy
from baybe_b200.engine import AcqConfig, unpack_best
from baybe_b200.synthetic import numeric_grid_workload
from tests import nei_oracle as no
from tests.helpers import oracle_model, posterior_tolerances

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
EPS32 = 2.0 ** -24


def test_joint_posterior_matches_a_float64_restatement():
    """The device normalises the fp32 rows with the fp32 bounds of bb_model and scales by its fp32 y statistics;
    everything else is float64, so the restatement with those same inputs agrees to 1e-9."""
    from oracle.reference_path import _kernel_diag, _standardised_posterior, kernel_matrix

    w = numeric_grid_workload(N=2000, d=6, n=96, seed=4)
    gp = DeviceGP(device=DEV, **w.gp_kwargs())
    om = oracle_model(w)
    rows = np.concatenate([w.train_x[:40], w.candidates[:50]]).astype(np.float32)
    mu, cov, (px, beta) = noisy._joint_posterior(gp, rows, with_beta=True)
    f32 = lambda v: torch.as_tensor(np.asarray(v, dtype=np.float32), dtype=torch.float64)  # noqa: E731
    Xn = (f32(rows) - f32(om.lo)) * f32(1.0 / om.rng.numpy())
    _, m, V = _standardised_posterior(om, Xn)
    c = kernel_matrix(om.spec, Xn, Xn) - V @ V.T
    c.diagonal().copy_(_kernel_diag(om.spec, Xn) - (V * V).sum(-1))
    ys, ym = float(np.float32(om.y_std)), float(np.float32(om.y_mean))
    ref_mu, ref_cov = ym + ys * m, ys * ys * c
    scale = ys * ys * float(om.spec.outputscale or 1.0)
    assert np.abs(mu - ref_mu.numpy()).max() <= 1e-9 * max(1.0, float(ref_mu.abs().max()))
    assert np.abs(cov - ref_cov.numpy()).max() <= 1e-9 * scale
    assert np.array_equal(cov, cov.T)
    assert (np.diag(cov)[:40] > 0).all()  # measured rows: variance near the noise level, still positive
    # beta from the same pass is what bb_pending_stats gives for the same rows (same kernel, same arithmetic)
    px31, beta31, _, _ = gp.pending_stats(rows[:31])
    assert torch.equal(beta[:31], beta31) and torch.equal(px[:31], px31)


def _recording(monkeypatch):
    seen = {}

    def rec(*args):
        seen["args"] = args
        return torch.ops.baybe_b200.nei_score(*args)

    monkeypatch.setattr(noisy, "_nei_score", rec)
    return seen


def _ref_and_bound(args):
    """Float64 value at the device's own inputs and a per-row bound derived from the fp32 error of the conditional
    moments: |L^-1 c|^2 and c . w are formed in fp32 from fp32 L^-1, c and w, so sigma^2 is off by at most
    e_r2 = 2 (C + 2) eps32 sum_j |r_j| (|L^-1| |c|)_j and the mean by e_m = (C + 2) eps32 max_s sum_j |c_j w_js| +
    eps32 |mu|; the bound is 2e-4 + 2e-4 |ref| (fp32 arithmetic of the reduction) plus twice the largest change of the
    float64 value over the corners (mu +- e_m, sigma^2 +- e_r2), as tests/helpers.score_bounds does."""
    mu, var, cross, linv, w, z, g, terms, _, log_nei, (a, b, tau_relu, tau_max), _, _ = args
    mu64, var64 = mu.double(), var.double()
    zx = z[:, -1].double()

    def value(m, v):
        return no.nei_values_f64(m, v, cross, linv, w, zx, g, terms, bool(log_nei), a, b, tau_relu, tau_max)

    ref = value(mu64, var64)
    C = 0 if cross is None else cross.shape[1]
    e_r2 = torch.zeros_like(mu64)
    e_m = EPS32 * mu64.abs()
    if C:
        c, L = cross.double(), linv.double()
        r = c @ L.T
        e_r2 = 2.0 * (C + 2) * EPS32 * (r.abs() * (c.abs() @ L.abs().T)).sum(1)
        e_m = e_m + (C + 2) * EPS32 * (c.abs() @ w.double().abs()).amax(1)
    e_r2 = e_r2 + 2 * EPS32 * var64.abs()
    dev = torch.zeros_like(ref)
    for sm in (-1.0, 1.0):
        for sv in (-1.0, 1.0):
            dev = torch.maximum(dev, (value(mu64 + sm * e_m, (var64 + sv * e_r2).clamp_min(0.0)) - ref).abs())
    return ref, 2e-4 + 2e-4 * ref.abs() + 2.0 * dev


def _workload(N=3000, n=40, seed=0, noise=1e-3):
    w = numeric_grid_workload(N=N, d=8, n=n, seed=seed)
    return dataclasses.replace(w, noise=np.array([noise]))


def _scorer(w, kind, n_base, prune=False):
    gp = DeviceGP(device=DEV, **w.gp_kwargs())
    cfg = AcqConfig(kind=kind, obj_scale=-1.3, obj_shift=0.2)
    return noisy.NeiScorer(gp, cfg, w.train_x[:n_base], prune=prune)


_CASES = [(kind, n_base, P, Q) for kind in ("qNEI", "qLogNEI")
          for (n_base, P, Q) in ((1, 0, 0), (4, 3, 0), (24, 5, 2), (1, 3, 3))]


@pytest.mark.parametrize("kind,n_base,P,Q", _CASES)
def test_device_matches_the_float64_definition_row_by_row(monkeypatch, kind, n_base, P, Q):
    """|C| = n_base + P + Q in {1, 7, 31} (|C| = 0 below), keep mask and index offset on the 7-point case."""
    w = _workload(seed=n_base + P)
    sc = _scorer(w, kind, n_base)
    X = w.candidates
    rng = np.random.default_rng(1)
    idx = rng.choice(len(X), P + Q, replace=False)
    pend, batch = (X[idx[:P]] if P else None), (X[idx[P:]] if Q else None)
    z = sc.base_samples(256, P + Q, seed=3)
    keep, off = None, 0
    if n_base + P + Q == 7:
        keep = torch.from_numpy((rng.random(len(X)) > 0.3).astype(np.uint8)).to(DEV)
        off = 12345
    seen = _recording(monkeypatch)
    s, key, _ = sc.values(torch.from_numpy(X), pend, z, keep=keep, index_offset=off, batch=batch)
    assert seen["args"][2].shape[1] == n_base + P + Q
    dev = s.double().cpu()
    ref, bound = _ref_and_bound(seen["args"])
    ref, bound = ref.cpu(), bound.cpu()
    err = (dev - ref).abs()
    assert not bool(torch.isnan(dev).any())
    assert bool((err <= bound).all()), f"max err {float(err.max()):.3e}, worst row {int((err - bound).argmax())}"
    assert int(key.item()) == int(sc.gp.argmax(s, keep, off).item())


@pytest.mark.parametrize("log_nei", [False, True])
def test_device_without_conditioning_points(log_nei):
    w = _workload()
    gp = DeviceGP(device=DEV, **w.gp_kwargs())
    mu, var = gp.posterior(torch.from_numpy(w.candidates))
    z = torch.randn(300, 1, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    g = torch.full((300,), float(mu.max()) - 0.05, dtype=torch.float64)
    args = (mu, var, None, None, None, z.to(DEV, torch.float32), g.to(DEV, torch.float32), None, None, log_nei,
            [1.0, 0.0, 1e-6, 1e-2], 0, True)
    s, key = torch.ops.baybe_b200.nei_score(*args)
    ref, bound = _ref_and_bound(args)
    assert bool(((s.double() - ref).abs() <= bound).all())
    assert unpack_best(int(key.item()))[1] == int(torch.argmax(s))


def test_greedy_batch_equals_the_oracle_greedy_batch(monkeypatch):
    from baybe_b200.recommenders import greedy_select

    w = _workload(N=2000, n=60, seed=5, noise=1e-2)
    sc = _scorer(w, "qLogNEI", 60, prune=True)
    X = w.candidates
    xd = torch.from_numpy(X).to(DEV, torch.float32)
    chosen, vals = greedy_select(sc, sc.cfg, xd, X.shape[1], 3, None, seed=9, n_samples=256)
    assert len(set(chosen)) == 3
    pend = np.zeros((0, X.shape[1]))
    for r in range(3):
        seen = _recording(monkeypatch)
        sc.values(torch.from_numpy(X), pend if len(pend) else None, sc.base_samples(256, len(pend), 9))
        ref, bound = (t.cpu() for t in _ref_and_bound(seen["args"]))
        ref[chosen[:r]] = -np.inf
        i_ref = int(torch.argmax(ref))
        assert i_ref == chosen[r] or float(ref[i_ref] - ref[chosen[r]]) <= float(bound[i_ref] + bound[chosen[r]])
        assert abs(float(ref[chosen[r]]) - vals[r]) <= float(bound[chosen[r]])
        pend = np.concatenate([pend, X[chosen[r]][None]])


def test_device_conditioning_agrees_with_the_oracle_posterior():
    """End to end against the float64 oracle: the device value of every row is within the bound that the stated
    posterior tolerances (tests/helpers.posterior_tolerances) of mu, sigma^2 and the cross covariance allow."""
    w = _workload(N=1500, n=40, seed=2, noise=1e-2)
    sc = _scorer(w, "qNEI", 40, prune=True)
    om = oracle_model(w)
    X = w.candidates[:800]
    z = sc.base_samples(256, 0, seed=5)
    s, _, _ = sc.values(torch.from_numpy(X), None, z)
    nc = sc.n_conditioning(0)
    rows = sc.baseline[sc.kept_baseline(0)]
    mu, var = oracle.posterior(om, X)
    m, cov = oracle.posterior_joint(om, np.concatenate([rows, X]))
    c = sc.cfg
    zz = z.numpy()
    mc, cc = m[:nc].numpy(), cov[:nc, :nc].numpy()
    L = np.linalg.cholesky(cc)
    linv = np.linalg.inv(L)
    g = (c.obj_scale * (mc[None] + zz[:, :nc] @ L.T) + c.obj_shift).max(1)
    cross = cov[nc:, :nc]

    def value(dm, dv, dc):
        return no.nei_values_f64(mu + dm, (var + dv).clamp_min(0), cross * (1 + dc), linv, (zz[:, :nc] @ linv).T,
                                 zz[:, nc], g, None, False, c.obj_scale, c.obj_shift, 1e-6, 1e-2)

    ref = value(0.0, 0.0, 0.0)
    dmu, dvar = posterior_tolerances(om, mu)
    dcr = dvar / float(cross.abs().max())
    dev = torch.zeros_like(ref)
    for a in (-1, 1):
        for b in (-1, 1):
            for e in (-1, 1):
                dev = torch.maximum(dev, (value(a * dmu, b * dvar, e * dcr) - ref).abs())
    bound = 2e-4 + 2e-4 * ref.abs() + 1.5 * dev
    err = (s.double().cpu() - ref).abs()
    assert bool((err <= bound).all()), f"max err {float(err.max()):.3e}, worst row {int((err - bound).argmax())}"


def test_one_million_candidates_qlognei(monkeypatch):
    """1M x 20D, n = 256, S = 512, qLogNEI with a pruned baseline: the device's recommended row is the float64
    definition's over all rows (same moments, conditioning and samples, float64 on the device)."""
    w = numeric_grid_workload(N=1_000_000, d=20, n=256, seed=0)
    gp = DeviceGP(device=DEV, **w.gp_kwargs())
    sc = noisy.NeiScorer(gp, AcqConfig(kind="qLogNEI"), w.train_x)
    z = sc.base_samples(512, 0, seed=1234)
    seen = _recording(monkeypatch)
    x32 = torch.from_numpy(w.candidates).to(DEV, torch.float32)
    s, key, _ = sc.values(x32, None, z)
    i_dev = unpack_best(int(key.item()))[1]
    assert i_dev == int(torch.argmax(s))
    args = list(seen["args"])
    ref = torch.empty(len(x32), dtype=torch.float64, device=DEV)
    step = 16384
    for c0 in range(0, len(x32), step):
        a = list(args)
        a[0], a[1], a[2] = args[0][c0:c0 + step], args[1][c0:c0 + step], args[2][c0:c0 + step]
        ref[c0:c0 + step] = no.nei_values_f64(a[0], a[1], a[2], a[3], a[4], a[5][:, -1], a[6], None, True,
                                              *args[10])
    i_ref = int(torch.argmax(ref))
    if i_dev != i_ref:  # only a tie within the stated bounds of the two rows is accepted
        a = list(args)
        a[0], a[1], a[2] = args[0][[i_dev, i_ref]], args[1][[i_dev, i_ref]], args[2][[i_dev, i_ref]]
        r2, b2 = _ref_and_bound(a)
        assert float(r2[1] - r2[0]) <= float(b2[0] + b2[1]), (i_dev, i_ref, float(ref[i_dev]), float(ref[i_ref]))


@pytest.mark.parametrize("kind", ["qNEI", "qLogNEI"])
def test_noisy_campaigns_on_the_device(kind):
    root = Path(__file__).resolve().parents[1]
    ref_dir = root / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(root / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe.acquisition import acqfs

    from baybe_b200 import baybe_plugin
    from tests.test_nei import check_noisy_flow, noisy_campaign

    acqf = {"qNEI": acqfs.qNoisyExpectedImprovement, "qLogNEI": acqfs.qLogNoisyExpectedImprovement}[kind]
    camp, space = noisy_campaign(baybe_plugin, acqf())
    check_noisy_flow(camp, space, np.random.default_rng(0), tol=1e-4)
    assert isinstance(camp.recommender._scorer, noisy.NeiScorer)
