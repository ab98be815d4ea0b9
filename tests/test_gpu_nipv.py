"""qNIPV on the device: bb_nipv_score row by row against the float64 definition (joint posterior of integration points,
candidates and conditioning points from the oracle, noisy Gaussian conditioning), the arg-max, determinism, large
runs and the supported range."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import DeviceGP
from baybe_b200.engine import AcqConfig, unpack_best
from baybe_b200.nipv import NipvScorer
from baybe_b200.synthetic import fingerprint_workload, numeric_grid_workload, task_workload
from tests.helpers import oracle_model

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _noise_orig(om, rows):
    noise = om.noise.numpy()
    if om.spec.task_idx is None:
        return np.full(len(rows), max(float(noise[0]), 1e-4)) * om.y_std**2
    t = np.clip(np.rint(rows[:, om.spec.task_idx]).astype(int), 0, len(noise) - 1)
    return np.maximum(noise[t], 1e-4) * om.y_std**2


def ivr64(om, X, XM, XC, chunk=4096):
    """IVR(x) = sum_m k_C(m,x)^2 / (k_C(x,x) + noise(x)) in original units, float64, from the joint posterior of
    [XM chunk; X; XC] conditioned on noisy observations of XC (the integration points in chunks)."""
    num, den = 0.0, None
    N, C = len(X), len(XC)
    for m0 in range(0, len(XM), chunk):
        xm = XM[m0:m0 + chunk]
        M = len(xm)
        rows = np.concatenate([xm, X, XC]).astype(np.float32).astype(np.float64)
        _, cov = oracle.posterior_joint(om, rows)
        cov = cov.numpy() if torch.is_tensor(cov) else np.asarray(cov)
        if C:
            c = slice(M + N, M + N + C)
            Kc = cov[c, c] + np.diag(_noise_orig(om, rows[c]))
            cov = cov - cov[:, c] @ np.linalg.solve(Kc, cov[c, :])
        num = num + (cov[M:M + N, :M] ** 2).sum(1)
        if den is None:
            den = np.diag(cov)[M:M + N] + _noise_orig(om, rows[M:M + N])
    return num / den


def _scorer(w, XM):
    gp = DeviceGP(device=DEV, **w.gp_kwargs())
    return gp, NipvScorer(gp, AcqConfig(kind="qNIPV"), XM)


def _check(w, X, XM, pend, keep=None, index_offset=0):
    gp, sc = _scorer(w, XM)
    om = oracle_model(w)
    kt = None if keep is None else torch.from_numpy(keep.astype(np.uint8)).to(DEV)
    s, key, _ = sc.values(X, pend, None, kt, index_offset)
    s = s.double().cpu().numpy()
    ref = ivr64(om, X, XM, np.zeros((0, X.shape[1])) if pend is None else pend)
    assert np.abs(s - ref).max() <= 2e-4 * ref.max(), (np.abs(s - ref).max(), ref.max())
    elig = np.ones(len(X), bool) if keep is None else keep.astype(bool)
    _, idx = unpack_best(int(key.item()))
    i = idx - index_offset
    assert elig[i]
    assert ref[i] >= ref[elig].max() * (1 - 1e-4)
    s2, key2, _ = sc.values(X, pend, None, kt, index_offset, want_scores=False)
    assert s2 is None and int(key2.item()) == int(key.item())
    s3, key3, _ = sc.values(X, pend, None, kt, index_offset)
    assert torch.equal(s3.cpu(), torch.from_numpy(s.astype(np.float32))) and int(key3.item()) == int(key.item())
    return s, ref


@pytest.mark.parametrize("family", ["matern12", "matern32", "matern52", "rbf"])
@pytest.mark.parametrize("n,d,C", [(16, 3, 0), (100, 20, 5), (256, 20, 31), (100, 62, 5)])
def test_ivr_matches_float64(family, n, d, C):
    w = numeric_grid_workload(N=700, d=d, n=n, seed=n + d, family=family)
    rng = np.random.default_rng(C)
    X = w.candidates[rng.choice(700, 333, replace=False)]
    XM = w.candidates[rng.choice(700, 197, replace=False)]
    pend = w.candidates[rng.choice(700, C, replace=False)] if C else None
    _check(w, X, XM, pend)


def test_task_model_keep_offset_and_single_integration_point():
    w = task_workload(N_per_task=150, n_tasks=3, d_num=6, n_per_task=40)
    rng = np.random.default_rng(1)
    X = w.candidates[rng.choice(len(w.candidates), 257, replace=False)]
    keep = rng.random(257) > 0.3
    _check(w, X, w.candidates[:1], w.candidates[5:8], keep=keep, index_offset=1000)
    _check(w, X, w.candidates[10:139], None)


def test_ties_go_to_the_lowest_index():
    w = numeric_grid_workload(N=300, d=4, n=30, seed=3)
    X = np.repeat(w.candidates[:3], 50, axis=0)
    gp, sc = _scorer(w, w.candidates[100:200])
    s, key, _ = sc.values(X, None, None)
    _, idx = unpack_best(int(key.item()))
    best = int(np.argmax(s.cpu().numpy()))
    assert idx == best and idx % 50 == 0


def test_large_1m_rows_4096_integration_points():
    w = numeric_grid_workload(N=1_000_000, d=20, n=256, seed=0)
    rng = np.random.default_rng(0)
    XM = w.candidates[rng.choice(len(w.candidates), 4096, replace=False)]
    pend = w.candidates[rng.choice(len(w.candidates), 8, replace=False)]
    gp, sc = _scorer(w, XM)
    s, key, _ = sc.values(w.candidates, pend, None)
    s = s.double().cpu().numpy()
    top = np.argsort(-s)[:1024]
    rows = np.unique(np.concatenate([top, rng.choice(len(s), 1024, replace=False)]))
    om = oracle_model(w)
    ref = np.concatenate([ivr64(om, w.candidates[r], XM, pend) for r in np.array_split(rows, 8)])
    assert np.abs(s[rows] - ref).max() <= 2e-4 * ref.max()
    _, idx = unpack_best(int(key.item()))
    assert idx == int(np.argmax(s))


def test_large_full_fraction_200k():
    w = numeric_grid_workload(N=200_000, d=20, n=256, seed=1)
    gp, sc = _scorer(w, w.candidates)
    s, key, _ = sc.values(w.candidates, None, None)
    s = s.double().cpu().numpy()
    rows = np.random.default_rng(2).choice(len(s), 256, replace=False)
    ref = ivr64(oracle_model(w), w.candidates[rows], w.candidates, np.zeros((0, 20)))
    assert np.abs(s[rows] - ref).max() <= 2e-4 * ref.max()


def test_several_workspace_blocks_of_candidates_and_integration_points(monkeypatch):
    """A workspace of a few hundred KB splits both sets into several row blocks: the integration points' tiles are
    rebuilt for every candidate block and the row sums are carried across the integration blocks."""
    from baybe_b200 import engine

    monkeypatch.setattr(engine, "_NIPV_WS_CAP", 300 << 10)  # 128 candidate rows, 256 integration rows per block
    w = numeric_grid_workload(N=1500, d=20, n=100, seed=9)
    rng = np.random.default_rng(4)
    X = w.candidates[rng.choice(1500, 333, replace=False)]
    XM = w.candidates[rng.choice(1500, 600, replace=False)]
    pend = w.candidates[rng.choice(1500, 5, replace=False)]
    split, _ = _check(w, X, XM, pend, index_offset=7)
    monkeypatch.setattr(engine, "_NIPV_WS_CAP", 768 << 20)
    whole = _scorer(w, XM)[1].values(X, pend, None)[0].double().cpu().numpy()
    assert np.abs(split - whole).max() <= 1e-5 * whole.max()


def test_outside_the_supported_range_raises():
    w = numeric_grid_workload(N=600, d=4, n=300, seed=2)
    gp = DeviceGP(device=DEV, **w.gp_kwargs())
    with pytest.raises(NotImplementedError, match="at most 256"):
        NipvScorer(gp, AcqConfig(kind="qNIPV"), w.candidates[:10])
    wf = fingerprint_workload(N=200, d=2048, n=64)
    gpw = DeviceGP(device=DEV, **wf.gp_kwargs())
    assert gpw.model.wide
    with pytest.raises(NotImplementedError, match="wide-feature"):
        NipvScorer(gpw, AcqConfig(kind="qNIPV"), wf.candidates[:10])


def test_nipv_campaign_on_the_device():
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

    camp, space = noisy_campaign(baybe_plugin, acqfs.qNegIntegratedPosteriorVariance())
    vals = check_noisy_flow(camp, space, np.random.default_rng(0), tol=1e-4)
    assert isinstance(camp.recommender._scorer, NipvScorer) and (vals < 0).all()
    fps = acqfs.qNegIntegratedPosteriorVariance(sampling_n_points=17, sampling_method="FPS")
    camp2, space2 = noisy_campaign(baybe_plugin, fps)
    from tests.test_mo import measure

    camp2.add_measurements(measure(space2.discrete.exp_rep.sample(12, random_state=1), np.random.default_rng(0),
                                   ("yield",)))
    assert len(camp2.recommend(batch_size=2)) == 2
    assert np.isfinite(camp2.acquisition_values(space2.discrete.exp_rep.head(15)).to_numpy()).all()
    assert np.isfinite(camp2.joint_acquisition_value(space2.discrete.exp_rep.head(2)))
