"""qLogNParEGO on the device: bb_parego_score row by row against the float64 definition of tests/parego_oracle.py fed
with the same moments, conditioning and base samples (M = 2, 5, 8; |C| = 1, 9, 31; S = 512, 1024; with and without
batch terms; keep mask and index offset), the 1M-row recommendation and real Campaign runs."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from baybe_b200 import DeviceGP, parego
from baybe_b200.engine import AcqConfig, unpack_best
from baybe_b200.synthetic import numeric_grid_workload, smooth_target
from tests import parego_oracle as po

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
EPS32 = 2.0 ** -24


def _recording(monkeypatch):
    seen = {}

    def rec(*args):
        seen["args"] = args
        return torch.ops.baybe_b200.parego_score(*args)

    monkeypatch.setattr(parego, "_parego_score", rec)
    return seen


def _ref_and_bound(args):
    """Float64 value at the device's own inputs (the fp32 weights and offsets included) and a per-row bound derived
    from the fp32 error of the conditional moments, as tests/test_gpu_nei._ref_and_bound does per target: sigma_m^2 is
    off by at most e_r2 = 2 (C + 2) eps32 sum_j |r_j| (|L^-1| |c|)_j + 2 eps32 var and the mean by
    e_m = (C + 2) eps32 max_s sum_j |c_j w_js| + eps32 |mu|; forming p_m, cheb and cheb - g in fp32 moves the
    improvement by at most e_u = (2M + 4) eps32 (max|g| + sum_m (|W_m| (|mu_m| + 6 sd_m + e_m') + |V_m|)).  The bound
    is 2e-4 + 2e-4 |ref| (fp32 arithmetic of the reduction) plus twice the largest change of the float64 value over
    the corners (mu +- e_m, sigma^2 +- e_r2, cheb - g +- e_u)."""
    mu, var, cross, linv, w, z, g, terms, _, W, V, (alpha, tau_relu, tau_max), _, _ = args
    W32 = np.float32(np.asarray(W, dtype=np.float64)).astype(np.float64)
    V32 = np.float32(np.asarray(V, dtype=np.float64)).astype(np.float64)
    M, N = mu.shape
    nc = 0 if cross is None else cross.shape[2]
    zx = torch.stack([z[:, m * (nc + 1) + nc] for m in range(M)], 1).double()
    mu64, var64, g64 = mu.double(), var.double(), g.double()

    def value(m_, v_, du=None):
        return po.parego_values_f64(m_, v_, cross, linv, w, zx, g64, terms, W32, V32, alpha, tau_relu, tau_max, du=du)

    ref = value(mu64, var64)
    e_m = EPS32 * mu64.abs()
    e_r2 = 2 * EPS32 * var64.abs()
    cw = torch.zeros_like(mu64)
    if nc:
        c, L = cross.double(), linv.double()
        r = torch.einsum("mnc,mkc->mnk", c, L)
        e_r2 = e_r2 + 2.0 * (nc + 2) * EPS32 * (r.abs() * torch.einsum("mnc,mkc->mnk", c.abs(), L.abs())).sum(2)
        cw = torch.einsum("mnc,mcs->mns", c.abs(), w.double().abs()).amax(2)
        e_m = e_m + (nc + 2) * EPS32 * cw
    Wt = torch.as_tensor(np.abs(W32), dtype=torch.float64, device=mu.device)[:, None]
    Vt = torch.as_tensor(np.abs(V32), dtype=torch.float64, device=mu.device)[:, None]
    mag = (Wt * (mu64.abs() + 6.0 * var64.clamp_min(0).sqrt() + cw) + Vt).sum(0)  # [N]
    e_u = (2 * M + 4) * EPS32 * (float(g64.abs().max()) + mag)
    dev = torch.zeros_like(ref)
    for sm in (-1.0, 1.0):
        for sv in (-1.0, 1.0):
            for su in (-1.0, 1.0):
                val = value(mu64 + sm * e_m, (var64 + sv * e_r2).clamp_min(0.0), su * e_u)
                dev = torch.maximum(dev, (val - ref).abs())
    return ref, 2e-4 + 2e-4 * ref.abs() + 2.0 * dev


def _models(M, n, seed=0, N=3000, noise=1e-3):
    w = numeric_grid_workload(N=N, d=8, n=n, seed=seed)
    kw = w.gp_kwargs()
    kw["noise"] = np.array([noise])
    gps = [DeviceGP(device=DEV, **{**kw, "train_y": smooth_target(w.train_x, seed=seed + 7 * m + 1)})
           for m in range(M)]
    return w, gps


def _scorer(w, gps, n_base, prune=False):
    M = len(gps)
    a = np.array([1.0, -1.0] * (M // 2) + [1.0] * (M % 2))
    lam = np.linspace(1.0, 2.0, M) / np.linspace(1.0, 2.0, M).sum()
    return parego.ParegoScorer(gps, AcqConfig(kind="qLogNParEGO"), a, np.linspace(0.0, 0.5, M), w.train_x[:n_base],
                               lam, prune=prune)


# (M, n_base, P, Q, S): |C| = n_base + P + Q
_CASES = [(2, 1, 0, 0, 512), (2, 1, 5, 3, 1024), (5, 4, 3, 2, 1024), (5, 31, 0, 0, 512), (8, 1, 0, 0, 1024),
          (8, 24, 5, 2, 512), (8, 9, 0, 0, 1024), (5, 1, 0, 0, 512)]


@pytest.mark.parametrize("M,n_base,P,Q,S", _CASES)
def test_device_matches_the_float64_definition_row_by_row(monkeypatch, M, n_base, P, Q, S):
    w, gps = _models(M, max(n_base, 8), seed=n_base + P)
    sc = _scorer(w, gps, n_base)
    X = w.candidates
    rng = np.random.default_rng(1)
    idx = rng.choice(len(X), P + Q, replace=False)
    pend, batch = (X[idx[:P]] if P else None), (X[idx[P:]] if Q else None)
    z = sc.base_samples(S, P + Q, seed=3)
    keep, off = None, 0
    if n_base + P + Q == 9:
        keep = torch.from_numpy((rng.random(len(X)) > 0.3).astype(np.uint8)).to(DEV)
        off = 12345
    seen = _recording(monkeypatch)
    s, key, _ = sc.values(torch.from_numpy(X), pend, z, keep=keep, index_offset=off, batch=batch)
    args = seen["args"]
    assert args[2].shape == (M, len(X), n_base + P + Q) and args[5].shape == (S, M * (n_base + P + Q + 1))
    dev = s.double().cpu()
    ref, bound = (t.cpu() for t in _ref_and_bound(args))
    err = (dev - ref).abs()
    assert not bool(torch.isnan(dev).any())
    assert bool((err <= bound).all()), f"max err {float(err.max()):.3e}, worst row {int((err - bound).argmax())}"
    assert int(key.item()) == int(gps[0].argmax(s, keep, off).item())


def test_device_without_conditioning_points():
    w, gps = _models(3, 20)
    mu, var = (torch.stack(t) for t in zip(*[gp.posterior(torch.from_numpy(w.candidates)) for gp in gps]))
    z = torch.randn(300, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    g = torch.full((300,), 0.2, dtype=torch.float64)
    args = (mu, var, None, None, None, z.to(DEV, torch.float32), g.to(DEV, torch.float32), None, None,
            [0.3, -0.2, 0.25], [-0.1, 0.9, 0.0], [0.05, 1e-6, 1e-2], 0, True)
    s, key = torch.ops.baybe_b200.parego_score(*args)
    ref, bound = _ref_and_bound(args)
    assert bool(((s.double() - ref).abs() <= bound).all())
    assert unpack_best(int(key.item()))[1] == int(torch.argmax(s))


def test_one_million_candidates_three_targets(monkeypatch):
    """1M x 20D, n = 256, S = 512, three targets, pruned baseline: the device's recommended row is the float64
    definition's over all rows (same moments, conditioning and samples, float64 on the device)."""
    w = numeric_grid_workload(N=1_000_000, d=20, n=256, seed=0)
    kw = w.gp_kwargs()
    gps = [DeviceGP(device=DEV, **{**kw, "train_y": smooth_target(w.train_x, seed=7 * m + 1)}) for m in range(3)]
    sc = parego.ParegoScorer(gps, AcqConfig(kind="qLogNParEGO"), np.array([1.0, -1.0, 1.0]), np.zeros(3),
                             w.train_x, np.array([0.2, 0.5, 0.3]))
    z = sc.base_samples(512, 0, seed=1234)
    seen = _recording(monkeypatch)
    x32 = torch.from_numpy(w.candidates).to(DEV, torch.float32)
    s, key, _ = sc.values(x32, None, z)
    i_dev = unpack_best(int(key.item()))[1]
    assert i_dev == int(torch.argmax(s))
    args = list(seen["args"])
    nc = args[2].shape[2]
    zx = torch.stack([args[5][:, m * (nc + 1) + nc] for m in range(3)], 1).double()
    W32 = np.float32(args[9]).astype(np.float64)
    V32 = np.float32(args[10]).astype(np.float64)
    ref = torch.empty(len(x32), dtype=torch.float64, device=DEV)
    step = 16384
    for c0 in range(0, len(x32), step):
        sl = slice(c0, c0 + step)
        ref[sl] = po.parego_values_f64(args[0][:, sl], args[1][:, sl], args[2][:, sl], args[3], args[4], zx, args[6],
                                       None, W32, V32, *args[11])
    i_ref = int(torch.argmax(ref))
    if i_dev != i_ref:  # only a tie within the stated bounds of the two rows is accepted
        a = list(args)
        rows = [i_dev, i_ref]
        a[0], a[1], a[2] = args[0][:, rows], args[1][:, rows], args[2][:, rows]
        r2, b2 = _ref_and_bound(a)
        assert float(r2[1] - r2[0]) <= float(b2[0] + b2[1]), (i_dev, i_ref, float(ref[i_dev]), float(ref[i_ref]))


@pytest.mark.parametrize("n_targets", [2, 5])
def test_parego_campaigns_on_the_device(monkeypatch, n_targets):
    root = Path(__file__).resolve().parents[1]
    ref_dir = root / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(root / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401

    from baybe_b200 import baybe_plugin
    from tests.test_parego import check_parego_flow

    camp = check_parego_flow(baybe_plugin, monkeypatch, n_targets, tol=1e-4)
    assert isinstance(camp.recommender._scorer, parego.ParegoScorer)
