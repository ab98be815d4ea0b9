"""Continuous and hybrid recommendation with the single-target acquisition functions (qLogEI, qEI, qUCB, qSR, qPI and the
analytic kinds) -- SURVEY.md 8f-2, the gradient path.

Replaces ``optimize_acqf`` for continuous spaces (``/root/reference/baybe/recommenders/pure/bayesian/botorch/
continuous.py:131-212``) and ``optimize_acqf_mixed`` for hybrid spaces (``botorch/hybrid.py:30-161``).  One routine
serves both: a continuous space is a hybrid space with one empty discrete configuration.

  * Raw stage: ``n_raw_samples`` scrambled-Sobol points in the continuous box, paired with every discrete
    configuration and scored in one sweep of the engine's scoring path (``recommenders._scores_for``, with the pending
    points).
  * Starts: ``n_restarts`` rows chosen as botorch's ``initialize_q_batch`` does [U]: Boltzmann weights
    exp(eta * standardised value), eta = 1, drawn without replacement by a seeded generator, the best raw row always
    included.  A hybrid start keeps its discrete configuration.
  * Polish: ``scipy.optimize.minimize(method="L-BFGS-B", jac=True)`` over the stacked starts on -sum(value), as
    botorch's ``gen_candidates_scipy`` stacks its restarts (maxiter 200 [U]); value and gradient come from
    ``bb_acq_grad``, or ``bb_acq_grad_large`` for wide models and n_pad > 256 (up to 1024 training points, chosen by
    ``engine.acq_grad_op``), one call over all starts per evaluation.  Fixed continuous parameters and discrete columns are not
    variables.  The best start wins, judged by the scoring path.
  * q > 1: sequential greedy (``optimize_acqf(sequential=True)``, ``optimize_acqf_mixed``): step j optimises the q = 1
    value given pending = [pending experiments; x_1 ... x_{j-1}].

Objectives that are not affine in their targets (desirability, transformed single targets) come as a
``baybe_b200.objectives.ObjectiveScorer`` in place of the model: raw and final values from its ``scores`` and
``joint_value``, gradients from its ``value_and_grad`` (``bb_objective_grad``, or ``bb_objective_grad_large`` when a target's
model is wide or has n_pad > 256, chosen by ``engine.objective_grad_op``), base samples of M(1+p) columns from its
``base_samples``.  Its pending-point conditioning is built once per greedy step and reused by every evaluation.
qNIPV comes the same way, as a ``baybe_b200.nipv.NipvScorer``: raw and final values from ``bb_nipv_score``, gradients
from ``bb_nipv_grad`` over the integration points' image, which is built once per greedy step with the conditioning
on [pending; earlier batch points].  qEHVI and qLogEHVI of Pareto objectives come as a
``baybe_b200.multiobjective.HviScorer``: raw and final values from ``bb_hvi_score``, gradients from ``bb_hvi_grad``;
the per-sample box decompositions of the front joined with the pending samples are built once per greedy step.

Deliberate deviation for hybrid spaces: the reference runs a full multi-start optimisation for every discrete
configuration (its own docstring calls that brute force).  Here the raw sweep ranks every configuration at once and the
``n_restarts`` best-placed starts are polished (DESIGN.md section 2).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.acquisition import AcqConfig
from baybe_b200.engine import sobol_normal_samples

__all__ = ["initial_starts", "recommend_continuous_hybrid", "MAXITER"]

MAXITER = 200  # botorch gen_candidates_scipy's L-BFGS-B default [U]
ETA = 1.0      # botorch initialize_q_batch's Boltzmann temperature [U]


def initial_starts(values: torch.Tensor, n: int, seed: int, eta: float = ETA) -> torch.Tensor:
    """Indices of ``n`` start rows out of raw rows with the given values (botorch ``initialize_q_batch`` [U])."""
    Y = torch.as_tensor(values, dtype=torch.float64).reshape(-1)
    Y = torch.where(torch.isfinite(Y), Y, torch.full_like(Y, -math.inf))
    N = Y.shape[0]
    if n >= N:
        return torch.arange(N)
    gen = torch.Generator().manual_seed(int(seed))
    finite = torch.isfinite(Y)
    if not bool(finite.any()):
        return torch.randperm(N, generator=gen)[:n]
    Yf = torch.where(finite, Y, Y[finite].min())
    std = Yf.std()
    if not bool(std > 0):
        idx = torch.randperm(N, generator=gen)[:n]
    else:
        Z = (Yf - Yf.mean()) / std
        w = torch.exp(eta * Z)
        while bool(torch.isinf(w).any()):
            eta *= 0.5
            w = torch.exp(eta * Z)
        idx = torch.multinomial(w, n, replacement=False, generator=gen)
    best = int(torch.argmax(Yf))
    if not bool((idx == best).any()):
        idx[-1] = best
    return idx


def _scores(gp, cfg: AcqConfig, rows: np.ndarray, pending: np.ndarray | None, seed: int, n_samples: int) -> np.ndarray:
    from baybe_b200.recommenders import _scores_for

    return _scores_for(gp, cfg, torch.from_numpy(np.ascontiguousarray(rows)), pending, seed,
                       n_samples).double().cpu().numpy()


def _is_scorer(gp) -> bool:
    """The scorers the gradient path serves in place of a model: ``ObjectiveScorer`` (desirability, transformed single
    targets), ``NipvScorer`` (qNIPV) and ``HviScorer`` (qEHVI / qLogEHVI)."""
    from baybe_b200.multiobjective import HviScorer
    from baybe_b200.nipv import NipvScorer
    from baybe_b200.objectives import ObjectiveScorer

    return isinstance(gp, (ObjectiveScorer, NipvScorer, HviScorer))


def _models(gp, scorer: bool) -> list:
    """The models behind `gp`: an ``ObjectiveScorer``'s or ``HviScorer``'s one per target, a ``NipvScorer``'s one, or
    `gp` itself."""
    if not scorer:
        return [gp]
    return list(gp.gps) if hasattr(gp, "gps") else [gp.gp]


def _polish(gp, cfg: AcqConfig, starts: np.ndarray, free: np.ndarray, lo: np.ndarray, hi: np.ndarray,
            pending: np.ndarray | None, z: torch.Tensor | None, stats: dict | None) -> np.ndarray:
    """L-BFGS-B over the free columns of the stacked starts on -sum(value); returns the final rows.  `gp`: a model
    (``value_and_grad(cfg, x, z, pending)``) or a scorer (``value_and_grad(x, pending, z)``)."""
    scorer = _is_scorer(gp)
    import time

    from scipy.optimize import minimize

    k, nf = starts.shape[0], len(free)
    base = starts.copy()

    def fg(v: np.ndarray):
        t0 = time.perf_counter()
        X = base.copy()
        X[:, free] = v.reshape(k, nf)
        if scorer:
            val, grad = gp.value_and_grad(torch.from_numpy(X.astype(np.float32)), pending, z)
        else:
            val, grad = gp.value_and_grad(cfg, torch.from_numpy(X.astype(np.float32)), z, pending)
        val = np.nan_to_num(val.double().cpu().numpy(), nan=0.0)
        g = np.nan_to_num(grad.double().cpu().numpy()[:, free], nan=0.0)
        if stats is not None:
            stats["grad_s"] = stats.get("grad_s", 0.0) + time.perf_counter() - t0
            stats["grad_calls"] = stats.get("grad_calls", 0) + 1
        return -float(val.sum()), -g.reshape(-1)

    bounds = list(zip(np.tile(lo, k), np.tile(hi, k)))
    t0 = time.perf_counter()
    res = minimize(fg, base[:, free].reshape(-1), jac=True, method="L-BFGS-B", bounds=bounds,
                   options={"maxiter": MAXITER})
    if stats is not None:
        stats["polish_s"] = stats.get("polish_s", 0.0) + time.perf_counter() - t0
    out = base.copy()
    out[:, free] = np.clip(res.x.reshape(k, nf), lo, hi)
    return out


def recommend_continuous_hybrid(gp, cfg: AcqConfig, disc_comp: np.ndarray, cont_bounds: np.ndarray,
                                batch_size: int, pending: np.ndarray | None = None, n_samples: int = 512,
                                seed: int = 0, n_raw_samples: int = 64, n_restarts: int = 10,
                                fixed: dict[int, float] | None = None, stats: dict | None = None):
    """Sequential-greedy batch over (discrete configurations) x (continuous box).  Returns (points
    [batch_size, d_disc + d_cont] float64 in comp-rep column order, discrete-configuration indices, joint value of
    [batch; pending]).

    ``disc_comp``: (n_configs, d_disc) comp-rep rows of the discrete subspace, which comes first in the comp-rep (a
    continuous space: one row of width 0); ``cont_bounds``: (2, d_cont); ``fixed``: continuous column -> value of the
    fixed parameters.  ``gp``: a ``DeviceGP`` (or a stand-in with ``value_and_grad``, ``score``, ``score_joint``), or an
    ``ObjectiveScorer``, ``NipvScorer`` or ``HviScorer`` (then ``cfg`` is its ``cfg``)."""
    scorer = _is_scorer(gp)
    kinds = _lib.GRAD_KINDS + (_lib.NIPV_KINDS + _lib.HVI_KINDS if scorer else ())
    if cfg.kind not in kinds:
        raise NotImplementedError(f"the gradient path serves {kinds}, not {cfg.kind!r}")
    if any(getattr(m, "task_col", None) is not None for m in _models(gp, scorer)):
        raise NotImplementedError("the gradient path supports single-task models")
    disc = np.asarray(disc_comp, dtype=np.float64).reshape(len(disc_comp), -1)
    cb = np.asarray(cont_bounds, dtype=np.float64)
    nc, dd, dc = disc.shape[0], disc.shape[1], cb.shape[1]
    pend0 = np.empty((0, dd + dc)) if pending is None else np.asarray(pending, dtype=np.float64).reshape(-1, dd + dc)
    if batch_size - 1 + len(pend0) > _lib.MAX_PENDING:
        raise NotImplementedError(f"batch_size - 1 + pending experiments must be at most {_lib.MAX_PENDING}")
    if batch_size > 1 and not cfg.is_mc:
        raise ValueError("analytic acquisition functions recommend one point at a time")
    fixed = dict(fixed or {})
    free_c = np.array([j for j in range(dc) if j not in fixed], dtype=np.int64)
    free = dd + free_c
    eng = torch.quasirandom.SobolEngine(dimension=max(dc, 1), scramble=True, seed=int(seed))
    u = eng.draw(n_raw_samples, dtype=torch.float64).numpy()[:, :dc]
    pts = cb[0] + u * (cb[1] - cb[0])
    for j, v in fixed.items():
        pts[:, j] = v
    rows = np.concatenate([np.repeat(disc, n_raw_samples, axis=0), np.tile(pts, (nc, 1))], axis=1)
    chosen, idx = [], []
    for step in range(batch_size):
        pend = np.vstack([pend0] + chosen)
        p = len(pend)
        if scorer:
            z = gp.base_samples(n_samples, p, seed)
            raw = gp.scores(rows, pend if p else None, seed, n_samples)
        else:
            z = sobol_normal_samples(n_samples, 1 + p, seed) if cfg.is_mc else None
            raw = _scores(gp, cfg, rows, pend if p else None, seed, n_samples)
        start_idx = initial_starts(torch.from_numpy(raw), n_restarts, seed + 1 + step).numpy()
        starts = rows[start_idx]
        if len(free):
            polished = _polish(gp, cfg, starts, free, cb[0, free_c], cb[1, free_c], pend if p else None, z, stats)
            cand = np.vstack([polished, starts])
        else:
            cand = starts
        if scorer:
            val = gp.scores(cand, pend if p else None, seed, n_samples)
        else:
            val = _scores(gp, cfg, cand, pend if p else None, seed, n_samples)
        val = np.where(np.isfinite(val), val, -np.inf)
        best = int(np.argmax(val))
        row = cand[best].copy()
        k = int(start_idx[best % len(start_idx)] // n_raw_samples)
        row[:dd] = disc[k]
        chosen.append(row[None])
        idx.append(k)
    batch = np.vstack(chosen)
    rest = np.vstack([batch[1:], pend0])
    if scorer:
        return batch, idx, gp.joint_value(batch, pend0 if len(pend0) else None, seed, n_samples)
    if len(rest):
        zj = sobol_normal_samples(n_samples, 1 + len(rest), seed)
        value = float(gp.score_joint(cfg, torch.from_numpy(batch[:1]), rest, zj)[0])
    else:
        value = float(_scores(gp, cfg, batch[:1], None, seed, n_samples)[0])
    return batch, idx, value
