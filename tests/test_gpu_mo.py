"""bb_hvi_score on the device (qEHVI / qLogEHVI for Pareto objectives) against the float64 definitions of
tests/mo_oracle.py and the stand-in of tests/test_mo.py."""
from __future__ import annotations

import dataclasses

import numpy as np
import pytest
import torch

import oracle
from baybe_b200 import DeviceGP, multiobjective as mo
from baybe_b200.engine import AcqConfig, unpack_best
from baybe_b200.synthetic import numeric_grid_workload, smooth_target
from tests import mo_oracle
from tests.helpers import oracle_model, posterior_tolerances
from tests.test_mo import _hvi_score_f64

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ORIENT = {2: ([1.0, -1.0], [0.0, 2.0]), 3: ([1.0, -1.0, 0.5], [0.0, 2.0, -1.0])}  # mixed orientation


def _workloads(M, N, n, seed=0, d=8):
    w0 = numeric_grid_workload(N=N, d=d, n=n, seed=seed)
    ws = [w0]
    for m in range(1, M):
        ws.append(dataclasses.replace(w0, train_y=smooth_target(w0.train_x, seed=20 + m)
                                      + 0.01 * np.random.default_rng(m).standard_normal(len(w0.train_y))))
    return ws


def _scorer(ws, kind):
    gps = [DeviceGP(device=DEV, **w.gp_kwargs()) for w in ws]
    oms = [oracle_model(w) for w in ws]
    a, b = (np.asarray(v) for v in ORIENT[len(ws)])
    front = np.stack([gp.posterior(torch.from_numpy(ws[0].train_x))[0].double().cpu().numpy() for gp in gps], 1) * a + b
    ref = mo.compute_ref_point(front)
    return mo.HviScorer(gps, AcqConfig(kind=kind), a, b, ref, front), oms


def _recording(monkeypatch):
    seen = {}

    def rec(*args):
        seen["args"] = args
        return torch.ops.baybe_b200.hvi_score(*args)

    monkeypatch.setattr(mo, "_hvi_score", rec)
    return seen


def _f64(args, mu, var):
    a = list(args)
    a[0], a[1] = mu, var
    return _hvi_score_f64(*[t.cpu() if torch.is_tensor(t) else t for t in a])[0].double()


def _ref_and_bound(args, oms, X, pending: bool):
    """Float64 value of the kernel's definition at the oracle's posterior (same cells, samples and pending inputs as
    the recorded call) and a hard per-row bound: fp32 arithmetic plus 1.5x the change the stated posterior tolerance
    (tests/helpers.py::posterior_tolerances) of each target can cause at that row."""
    post = [oracle.posterior(om, X) for om in oms]
    mu = torch.stack([p[0] for p in post]).float()
    var = torch.stack([p[1] for p in post]).float()
    ref = _f64(args, mu, var)
    sens = torch.zeros_like(ref)
    for m, om in enumerate(oms):
        dmu, dvar = posterior_tolerances(om, post[m][0])
        for dm, dv in ((dmu, 0.0), (-dmu, 0.0), (0.0, dvar), (0.0, -dvar)):
            mu2, var2 = mu.clone(), var.clone()
            mu2[m] += dm
            var2[m] = (var2[m] + dv).clamp_min(1e-12)
            sens += (_f64(args, mu2, var2) - ref).abs() / 2.0
    return ref, 2e-4 + 1e-4 * ref.abs() + 1.5 * sens + (5e-4 * ref.abs() if pending else 0.0)


def _same_winner(i_dev: int, i_ref: int, ref, bound) -> bool:
    """The device's recommended row is the oracle's, unless the two rows' float64 values are closer than their
    bounds (a tie at the resolution the posterior tolerance allows)."""
    return i_dev == i_ref or float(ref[i_ref] - ref[i_dev]) <= float(bound[i_ref] + bound[i_dev])


@pytest.mark.parametrize("kind", ["qLogEHVI", "qEHVI"])
@pytest.mark.parametrize("M,P,n", [(2, 0, 30), (2, 0, 256), (3, 0, 256), (2, 1, 30), (2, 3, 256), (3, 3, 30)])
def test_device_matches_the_float64_definition_row_by_row(monkeypatch, kind, M, P, n):
    N = 20000 if P == 0 else 4000
    ws = _workloads(M, N, n, seed=M + P + n)
    scorer, oms = _scorer(ws, kind)
    X = ws[0].candidates
    rng = np.random.default_rng(1)
    pend = X[rng.choice(N, P, replace=False)] if P else None
    z = scorer.base_samples(128, P, seed=3)
    seen = _recording(monkeypatch)
    dev, key, report = scorer.values(torch.from_numpy(X), pend, z)
    dev = dev.double().cpu()
    ref, bound = _ref_and_bound(seen["args"], oms, X, P > 0)
    err = (dev - ref).abs()
    assert bool((err <= bound).all()), f"max err {float(err.max()):.3e}, worst row {int((err - bound).argmax())}"
    i_dev = unpack_best(int(key.item()))[1]
    assert i_dev == int(torch.argmax(dev))
    assert _same_winner(i_dev, int(torch.argmax(ref)), ref, bound), (i_dev, int(torch.argmax(ref)))
    # the fully independent evaluation (own joint posteriors, own pending samples) on the first rows
    full = mo_oracle.ehvi(oms, kind, scorer.a, scorer.b, scorer.ref, scorer.front, X[:256], pend, z)
    rep = torch.tensor([report(float(v)) for v in dev[:256]], dtype=torch.float64)
    assert bool(((rep - full).abs() <= bound[:256] + 1e-3 * full.abs()).all())


@pytest.mark.parametrize("kind", ["qLogEHVI", "qEHVI"])
def test_greedy_batch_equals_the_oracle_greedy_batch(kind):
    from baybe_b200.recommenders import greedy_select

    ws = _workloads(2, 2000, 30, seed=5)
    scorer, oms = _scorer(ws, kind)
    X = ws[0].candidates
    xd = torch.from_numpy(X).to(DEV, torch.float32)
    chosen, vals = greedy_select(scorer, scorer.cfg, xd, X.shape[1], 3, None, seed=9, n_samples=128)
    pend = np.zeros((0, X.shape[1]))
    for r in range(3):
        z = scorer.base_samples(128, len(pend), 9)
        v = mo_oracle.ehvi(oms, kind, scorer.a, scorer.b, scorer.ref, scorer.front, X, pend if len(pend) else None, z)
        v[chosen[:r]] = -np.inf
        top2 = torch.topk(v, 2).values
        # a near-tie within the float32 resolution may go either way; otherwise the winners are identical
        if float(top2[0] - top2[1]) > 1e-5 * max(1.0, abs(float(top2[0]))):
            assert int(torch.argmax(v)) == chosen[r]
        assert abs(float(v[chosen[r]]) - vals[r]) < 1e-3 * max(1.0, abs(vals[r]))
        pend = np.concatenate([pend, X[chosen[r]][None]])


def test_keep_mask_offsets_ties_and_ragged_rows():
    ws = _workloads(2, 1001, 30, seed=7)  # ragged: not a multiple of the 8 rows per block
    scorer, _ = _scorer(ws, "qLogEHVI")
    X = ws[0].candidates.copy()
    X[500] = X[700]  # identical rows: identical scores, the lower index wins
    z = scorer.base_samples(64, 0, 1)
    s, key, _ = scorer.values(torch.from_numpy(X), None, z)
    s = s.cpu()
    assert float(s[500]) == float(s[700])
    keep = torch.ones(len(X), dtype=torch.uint8, device=DEV)
    best = int(torch.argmax(s))
    keep[best] = 0
    if best != 500:
        keep[[i for i in range(len(X)) if float(s[i]) > float(s[500]) and i != best]] = 0
    _, key2, _ = scorer.values(torch.from_numpy(X), None, z, keep=keep, index_offset=12345)
    val, idx = unpack_best(int(key2.item()))
    masked = s.clone()
    masked[keep.cpu() == 0] = -np.inf
    assert idx - 12345 == int(torch.argmax(masked)) and val == float(masked.max())
    if best != 500:
        assert idx - 12345 == 500
    keep.zero_()
    _, key3, _ = scorer.values(torch.from_numpy(X), None, z, keep=keep)
    assert unpack_best(int(key3.item()))[1] == -1


def test_pending_decompositions_have_different_cell_counts(monkeypatch):
    ws = _workloads(2, 3000, 30, seed=11)
    scorer, oms = _scorer(ws, "qEHVI")
    X = ws[0].candidates
    pend = X[[3, 17, 400]]
    seen = _recording(monkeypatch)
    z = scorer.base_samples(128, 3, 2)
    dev, _, report = scorer.values(torch.from_numpy(X), pend, z)
    counts = seen["args"][8].cpu().numpy()
    assert counts.min() < counts.max()
    full = mo_oracle.ehvi(oms, "qEHVI", scorer.a, scorer.b, scorer.ref, scorer.front, X[:300], pend, z)
    rep = torch.tensor([report(float(v)) for v in dev[:300].double().cpu()], dtype=torch.float64)
    assert bool(((rep - full).abs() <= 1e-3 + 1e-3 * full.abs()).all())


def test_pareto_campaign_on_the_device(monkeypatch):
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parents[1]
    ref_dir = root / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(root / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe.acquisition.acqfs import qLogExpectedHypervolumeImprovement

    from baybe_b200 import baybe_plugin
    from tests.test_mo import check_subset_batch_wins, measure, pareto_campaign

    rng = np.random.default_rng(0)
    camp, space = pareto_campaign(baybe_plugin, qLogExpectedHypervolumeImprovement())
    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, rng))
    rec = camp.recommend(batch_size=3)
    assert len(rec) == 3 and rec.index.is_unique and not set(rec.index) & set(seed_rows.index)
    camp.add_measurements(measure(rec, rng))
    torch.manual_seed(4)
    r1 = camp.recommend(batch_size=1)
    torch.manual_seed(4)
    vals = camp.acquisition_values(space.discrete.exp_rep)
    remaining = vals.drop(index=list(seed_rows.index) + list(rec.index))
    assert float(vals.loc[r1.index[0]]) >= float(remaining.max()) - 1e-4 * max(1.0, abs(float(remaining.max())))
    check_subset_batch_wins(baybe_plugin, monkeypatch, np.random.default_rng(5), qLogExpectedHypervolumeImprovement())


def test_one_million_candidates_two_targets(monkeypatch):
    """1M x 20D, 2 targets, n = 256, S = 512, qLogEHVI: the device's recommended row is the float64 oracle's over
    all rows (posterior by the oracle in float64, the cell sums in float64 on the device in row chunks)."""
    w = numeric_grid_workload(N=1_000_000, d=20, n=256, seed=0)
    ws = [w, dataclasses.replace(w, train_y=smooth_target(w.train_x, seed=21)
                                 + 0.01 * np.random.default_rng(1).standard_normal(len(w.train_y)))]
    scorer, oms = _scorer(ws, "qLogEHVI")
    z = scorer.base_samples(512, 0, seed=1234)
    x32 = torch.from_numpy(w.candidates).to(DEV, torch.float32)
    dev_scores, key, _ = scorer.values(x32, None, z)
    i_dev = unpack_best(int(key.item()))[1]
    assert i_dev == int(torch.argmax(dev_scores))
    lo = torch.from_numpy(scorer.lower).to(DEV)
    up = torch.from_numpy(scorer.upper).to(DEV)
    zx = z.to(DEV)  # P = 0: column m is target m's candidate sample
    a = torch.from_numpy(scorer.a).to(DEV)
    b = torch.from_numpy(scorer.b).to(DEV)
    post = [oracle.posterior(om, w.candidates, chunk=32768) for om in oms]
    ref = torch.empty(len(w.candidates), dtype=torch.float64)
    step = 4096
    for c0 in range(0, len(ref), step):
        mu = torch.stack([p[0][c0:c0 + step] for p in post], -1).to(DEV)
        sd = torch.stack([p[1][c0:c0 + step] for p in post], -1).to(DEV).sqrt()
        Y = a * (mu[None] + sd[None] * zx[:, None, :]) + b  # (S, rows, M)
        v = mo_oracle.cell_values(Y, lo, up, log=True)
        ref[c0:c0 + step] = (torch.logsumexp(v, 0) - np.log(Y.shape[0])).cpu()
    i_ref = int(torch.argmax(ref))
    if i_dev != i_ref:  # only a tie within the stated bounds of the two rows is accepted
        seen = _recording(monkeypatch)
        scorer.values(torch.from_numpy(w.candidates[[i_dev, i_ref]]), None, z)
        r2, b2 = _ref_and_bound(seen["args"], oms, w.candidates[[i_dev, i_ref]], False)
        assert float(r2[1] - r2[0]) <= float(b2[0] + b2[1]), (i_dev, i_ref, float(ref[i_dev]), float(ref[i_ref]))
