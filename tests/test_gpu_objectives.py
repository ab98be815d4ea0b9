"""bb_objective_score on the device (desirability and non-affine single-target objectives) against the float64
definition of tests/objective_oracle.py, fed with the same posterior moments (bb_posterior) and base samples."""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import pytest
import torch

from baybe_b200 import DeviceGP, objectives as ob
from baybe_b200.engine import AcqConfig, unpack_best
from baybe_b200.synthetic import numeric_grid_workload, smooth_target
from tests import objective_oracle as oo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

# per-target programs in the compiled form: normalised ramp, bell, triangular, sigmoid, a composite, ...
_PROGS = [
    [("CLAMP", (-1.0, 1.5, 0.0)), ("AFFINE", (0.4, 0.4, 0.0))],
    [("BELL", (0.2, 0.8, 0.0))],
    [("TWO_SIDED", (2.0, -0.5, 0.3)), ("AFFINE", (1.0, 1.0, 0.0)), ("CLAMP", (0.0, math.inf, 0.0))],
    [("SIGMOID", (0.1, -3.0, 0.0))],
    [("EXP", (0, 0, 0)), ("DUP_INPUT", (0, 0, 0)), ("SIGMOID", (0.5, 2.0, 0.0)), ("MUL", (0, 0, 0)),
     ("CLAMP", (0.0, 1.0, 0.0))],
    [("AFFINE", (-1.0, 1.0, 0.0)), ("CLAMP", (0.0, 1.0, 0.0))],
    [("POW_INT", (2.0, 0, 0)), ("DUP_INPUT", (0, 0, 0)), ("BELL", (0.0, 1.0, 0.0)), ("ADD", (0, 0, 0)),
     ("AFFINE", (0.3, 0.0, 0.0)), ("CLAMP", (0.0, 1.0, 0.0))],
    [("TWO_SIDED", (-1.0, 1.0, 0.0)), ("AFFINE", (-0.5, 1.0, 0.0)), ("CLAMP", (0.0, 1.0, 0.0))],
]


def _workloads(M, N, n, seed=0, d=8):
    w0 = numeric_grid_workload(N=N, d=d, n=n, seed=seed)
    ws = [w0]
    for m in range(1, M):
        ws.append(dataclasses.replace(w0, train_y=smooth_target(w0.train_x, seed=20 + m)
                                      + 0.01 * np.random.default_rng(m).standard_normal(len(w0.train_y))))
    return ws


def _scorer(ws, kind, scal, beta=0.5):
    gps = [DeviceGP(device=DEV, **w.gp_kwargs()) for w in ws]
    M = len(gps)
    wts = np.arange(1.0, M + 1.0)
    comp = ob.CompiledObjective([f"t{m}" for m in range(M)], _PROGS[:M], "NONE" if M == 1 else scal, wts / wts.sum())
    means = np.stack([gp.posterior(torch.from_numpy(ws[0].train_x))[0].double().cpu().numpy() for gp in gps], 1)
    best_f = float(np.max(ob.evaluate_objective(comp, means)))
    return ob.ObjectiveScorer(gps, AcqConfig(kind=kind, best_f=best_f, beta=beta), comp)


def _recording(monkeypatch):
    seen = {}

    def rec(*args):
        seen["args"] = args
        return torch.ops.baybe_b200.objective_score(*args)

    monkeypatch.setattr(ob, "_objective_score", rec)
    return seen


def _f64(args, mu=None):
    a = [t.cpu() if torch.is_tensor(t) else t for t in args]
    if mu is not None:
        a[0] = mu
    return oo.objective_score_f64(*a)[0].double()


def _ref_and_bound(args):
    """Float64 value at the device's own moments and samples, and a per-row bound: fp32 arithmetic plus 2x the change
    an fp32 rounding of every sample (2^-22 relative to |mu| + 4 sd, through the local slope of the objective) can
    cause at that row."""
    mu = args[0].cpu().double()
    sd = args[1].cpu().double().clamp_min(0).sqrt()
    ref = _f64(args, mu.float())
    sens = torch.zeros_like(ref)
    for sgn in (-1.0, 1.0):
        d = sgn * 2.0 ** -22 * (mu.abs() + 4.0 * sd + 1e-3)
        sens = torch.maximum(sens, (_f64(args, (mu + d)) - ref).abs())
    return ref, 2e-4 + 2e-4 * ref.abs() + 2.0 * sens


_CASES = [(M, kind, scal, P) for (M, scal) in ((1, "NONE"), (2, "GEOM_MEAN"), (3, "MEAN"), (8, "GEOM_MEAN"))
          for kind in ("qLogEI", "qEI", "qPI", "qSR", "qUCB") for P in (0, 7)]
_CASES += [(2, "qLogEI", "GEOM_MEAN", 1), (2, "qEI", "MEAN", 31), (3, "qUCB", "GEOM_MEAN", 31),
           (8, "qLogEI", "MEAN", 1), (1, "qPI", "NONE", 31)]


@pytest.mark.parametrize("M,kind,scal,P", _CASES)
def test_device_matches_the_float64_definition_row_by_row(monkeypatch, M, kind, scal, P):
    N = 3000
    ws = _workloads(M, N, 30, seed=M + P)
    scorer = _scorer(ws, kind, scal)
    X = ws[0].candidates
    pend = X[np.random.default_rng(1).choice(N, P, replace=False)] if P else None
    z = scorer.base_samples(128, P, seed=3)
    seen = _recording(monkeypatch)
    dev, key, _ = scorer.values(torch.from_numpy(X), pend, z)
    dev = dev.double().cpu()
    ref, bound = _ref_and_bound(seen["args"])
    err = (dev - ref).abs()
    assert not bool(torch.isnan(dev).any())
    assert bool((err <= bound).all()), f"max err {float(err.max()):.3e}, worst row {int((err - bound).argmax())}"
    assert unpack_best(int(key.item()))[1] == int(torch.argmax(dev))


def test_greedy_batch_equals_the_oracle_greedy_batch(monkeypatch):
    from baybe_b200.recommenders import greedy_select

    ws = _workloads(2, 2000, 30, seed=5)
    scorer = _scorer(ws, "qLogEI", "GEOM_MEAN")
    X = ws[0].candidates
    xd = torch.from_numpy(X).to(DEV, torch.float32)
    chosen, vals = greedy_select(scorer, scorer.cfg, xd, X.shape[1], 3, None, seed=9, n_samples=128)
    pend = np.zeros((0, X.shape[1]))
    for r in range(3):
        seen = _recording(monkeypatch)
        z = scorer.base_samples(128, len(pend), 9)
        scorer.values(torch.from_numpy(X), pend if len(pend) else None, z)
        ref, bound = _ref_and_bound(seen["args"])
        ref[chosen[:r]] = -np.inf
        i_ref = int(torch.argmax(ref))
        assert i_ref == chosen[r] or float(ref[i_ref] - ref[chosen[r]]) <= float(bound[i_ref] + bound[chosen[r]])
        assert abs(float(ref[chosen[r]]) - vals[r]) <= float(bound[chosen[r]])
        pend = np.concatenate([pend, X[chosen[r]][None]])


def test_keep_mask_offsets_ties_and_ragged_rows():
    ws = _workloads(2, 1001, 30, seed=7)  # ragged: not a multiple of the 8 rows per block
    scorer = _scorer(ws, "qLogEI", "GEOM_MEAN")
    X = ws[0].candidates.copy()
    X[500] = X[700]  # identical rows: identical scores, the lower index wins
    z = scorer.base_samples(64, 0, 1)
    s, key, _ = scorer.values(torch.from_numpy(X), None, z)
    s = s.cpu()
    assert float(s[500]) == float(s[700])
    assert unpack_best(int(key.item()))[1] == unpack_best(int(scorer.gps[0].argmax(s.to(DEV), None).item()))[1]
    keep = torch.ones(len(X), dtype=torch.uint8, device=DEV)
    best = int(torch.argmax(s))
    keep[best] = 0
    if best != 500:
        keep[[i for i in range(len(X)) if float(s[i]) > float(s[500]) and i != best]] = 0
    _, key2, _ = scorer.values(torch.from_numpy(X), None, z, keep=keep, index_offset=12345)
    key_am = scorer.gps[0].argmax(s.to(DEV), keep, 12345)
    assert int(key2.item()) == int(key_am.item())
    if best != 500:
        assert unpack_best(int(key2.item()))[1] - 12345 == 500
    keep.zero_()
    _, key3, _ = scorer.values(torch.from_numpy(X), None, z, keep=keep)
    assert unpack_best(int(key3.item()))[1] == -1


def test_one_million_candidates_two_target_desirability(monkeypatch):
    """1M x 20D, n = 256, S = 512, qLogEI, GEOM_MEAN of a clamp-normalised and a triangular target: the device's
    recommended row is the float64 definition's over all rows (same moments and samples, float64 on the device)."""
    w = numeric_grid_workload(N=1_000_000, d=20, n=256, seed=0)
    ws = [w, dataclasses.replace(w, train_y=smooth_target(w.train_x, seed=21)
                                 + 0.01 * np.random.default_rng(1).standard_normal(len(w.train_y)))]
    scorer = _scorer(ws, "qLogEI", "GEOM_MEAN")
    scorer.comp.programs[1] = _PROGS[2]
    scorer.kernel_comp = scorer.comp
    z = scorer.base_samples(512, 0, seed=1234)
    seen = _recording(monkeypatch)
    x32 = torch.from_numpy(w.candidates).to(DEV, torch.float32)
    dev_scores, key, _ = scorer.values(x32, None, z)
    i_dev = unpack_best(int(key.item()))[1]
    assert i_dev == int(torch.argmax(dev_scores))
    mu, var = seen["args"][0].double(), seen["args"][1].double()
    zx = z.to(DEV)
    ref = torch.empty(mu.shape[1], dtype=torch.float64)
    step = 8192
    for c0 in range(0, mu.shape[1], step):
        Y = mu[:, c0:c0 + step].T[None] + var[:, c0:c0 + step].clamp_min(0).sqrt().T[None] * zx[:, None, :]
        o = oo.objective(scorer.comp.programs, "GEOM_MEAN", scorer.comp.weights, Y)
        ref[c0:c0 + step] = oo.values_from_samples("qLogEI", o, None, scorer.cfg.best_f, 0.2, 1e-6, 1e-2, 1e-3).cpu()
    i_ref = int(torch.argmax(ref))
    if i_dev != i_ref:  # only a tie within the stated bounds of the two rows is accepted
        args = list(seen["args"])
        args[0], args[1] = args[0][:, [i_dev, i_ref]], args[1][:, [i_dev, i_ref]]
        r2, b2 = _ref_and_bound(args)
        assert float(r2[1] - r2[0]) <= float(b2[0] + b2[1]), (i_dev, i_ref, float(ref[i_dev]), float(ref[i_ref]))


def test_desirability_and_triangular_campaigns_on_the_device():
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
    from baybe import Campaign
    from baybe.objectives import SingleTargetObjective
    from baybe.targets import NumericalTarget

    from baybe_b200 import baybe_plugin
    from baybe_b200.surrogates import GaussianProcessSurrogate
    from tests.test_mo import measure, pareto_campaign
    from tests.test_objectives import check_flow, desirability_campaign

    camp, space = desirability_campaign(baybe_plugin)
    check_flow(camp, space, np.random.default_rng(0), tol=1e-4)
    _, space = pareto_campaign(baybe_plugin, None)
    hp = {"lengthscale": np.full(len(space.comp_rep_columns), 0.9), "noise": 5e-3, "mean_const": 0.0}
    rec = baybe_plugin.B200BotorchRecommender(surrogate_model=GaussianProcessSurrogate(hyperparameters=hp),
                                              n_mc_samples=128)
    camp = Campaign(space, SingleTargetObjective(NumericalTarget.match_triangular("yield", cutoffs=(50.0, 60.0))),
                    rec, allow_recommending_already_measured=False)
    seed_rows = space.discrete.exp_rep.sample(12, random_state=1)
    camp.add_measurements(measure(seed_rows, np.random.default_rng(0), ("yield",)))
    torch.manual_seed(3)
    r1 = camp.recommend(batch_size=1)
    torch.manual_seed(3)
    vals = camp.acquisition_values(space.discrete.exp_rep).drop(index=seed_rows.index)
    assert float(vals.loc[r1.index[0]]) >= float(vals.max()) - 1e-4 * max(1.0, abs(float(vals.max())))
    assert len(camp.recommend(batch_size=3)) == 3
