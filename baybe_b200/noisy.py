"""Noisy expected improvement on discrete search spaces: qNoisyExpectedImprovement and qLogNoisyExpectedImprovement
(``/root/reference/baybe/acquisition/acqfs.py:226-243``; ``X_baseline`` = the measured rows,
``acquisition/_builder.py:319-324``).

The host owns what does not depend on the candidate, in float64:
  * the pruned baseline (botorch's ``prune_inferior_points``, ``prune_winners`` / ``kept_points``): the measured
    rows that are the best of at least one of 2048 joint posterior samples, from ``bb_joint_posterior``;
  * the conditioning set C = [kept baseline; pending; other points of a q-batch], its joint samples, the per-sample
    incumbent g_s (the hard maximum of the objective over baseline and pending points) and the per-sample terms of
    the other batch points.
``bb_nei_score`` (csrc/nei.cu) samples every candidate conditionally on C and reduces over the samples on the
device; the sequential-greedy loop is ``baybe_b200.recommenders.greedy_select``.  Pending points join C and the
incumbent (botorch's ``incremental=True``): a greedy round values the improvement over everything chosen so far.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.engine import AcqConfig, sobol_normal_samples
from baybe_b200.scoring import Scorer

__all__ = ["PRUNE_SAMPLES", "PRUNE_SEED", "prune_winners", "kept_points", "capped_baseline", "condition_on",
           "BaselineScorer", "NeiScorer", "build_nei_scorer"]

PRUNE_SAMPLES = 2048  # botorch prune_inferior_points' num_samples
# botorch draws the pruning samples from the global RNG; a fixed seed keeps the pruned baseline the same in every call
# on the same data, so that a recommendation and the acquisition values reported for it condition on the same points
PRUNE_SEED = 0


def _nei_score(*args):
    """``baybe_b200::nei_score`` (engine.py); a module-level seam so that CPU tests can put a float64 stand-in here."""
    return torch.ops.baybe_b200.nei_score(*args)


def _joint_posterior(gp, rows: np.ndarray, with_beta: bool = False):
    """Float64 posterior mean [R] and covariance [R, R] of raw comp-rep rows (``baybe_b200::joint_posterior``) and,
    with `with_beta`, from the same pass the (rows, beta) pair that ``DeviceGP.cross_covariance`` takes for them as
    conditioning points (else None); a module-level seam like ``_nei_score``."""
    x = torch.from_numpy(np.ascontiguousarray(rows, dtype=np.float32)).to(gp.device)
    mu, cov, beta = torch.ops.baybe_b200.joint_posterior(x, gp.handle, bool(with_beta))
    return mu.cpu().numpy(), cov.cpu().numpy(), ((x, beta) if with_beta else None)


def prune_winners(o: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """Rows that are the arg-max of at least one sample of o [samples, n] (ties go to the first index), in
    ascending order, and how many samples each wins."""
    return np.unique(np.argmax(o, axis=1), return_counts=True)


def kept_points(winners: np.ndarray, counts: np.ndarray, cap: int) -> np.ndarray:
    """The winners if at most `cap`, else the `cap` most frequent ones (stable sort by count, descending), returned
    in ascending index order."""
    if len(winners) <= cap:
        return winners
    return np.sort(winners[np.argsort(-counts, kind="stable")[:cap]])


def capped_baseline(name: str, winners: np.ndarray, counts: np.ndarray, n_rows: int, prune: bool,
                    n_other: int) -> tuple[np.ndarray, int]:
    """The baseline rows (indices into the `n_rows` measured rows) that condition an evaluation with `n_other`
    pending and batch points, and how many winners were left out: ``kept_points`` capped at ``MAX_PENDING`` -
    `n_other`; without pruning every row, or ``NotImplementedError`` if they do not fit."""
    cap = _lib.MAX_PENDING - n_other
    if not prune and n_rows > cap:
        raise NotImplementedError(
            f"{name} with prune_baseline=False conditions on all {n_rows} measured rows plus "
            f"{n_other} pending/batch points; the B200 engine conditions on at most {_lib.MAX_PENDING} points "
            "(BB_MAX_PENDING): use prune_baseline=True or fewer measurements")
    if cap < 1:
        raise NotImplementedError(
            f"{name} with {n_other} pending/batch points leaves no room for a baseline point; the B200 "
            f"engine conditions on at most {_lib.MAX_PENDING} points (BB_MAX_PENDING)")
    kept = kept_points(winners, counts, cap)
    return kept, len(winners) - len(kept)


def condition_on(gp, rows: np.ndarray):
    """Float64 posterior mean mu [R] of the conditioning rows under one model, the Cholesky factor L [R, R] of their
    covariance and L^-1, and the (rows, beta) pair ``cross_covariance`` takes for them."""
    from baybe_b200.multiobjective import _psd_cholesky

    mu, cov, cond = _joint_posterior(gp, rows, with_beta=True)
    L = _psd_cholesky(0.5 * (cov + cov.T))
    return mu, L, np.linalg.inv(L), cond


def _log_fatplus(u: np.ndarray, tau: float) -> np.ndarray:
    """log fatplus(u, tau) = log tau + log(softplus(u / tau) + 0.1 / (1 + (u / tau)^2)) (botorch, alpha = 0.1)."""
    t = u / tau
    return math.log(tau) + np.log(np.logaddexp(0.0, t) + 0.1 / (1.0 + t * t))


class BaselineScorer(Scorer):
    """A scorer over one model per target that conditions every evaluation on a baseline of measured rows (raw
    comp-rep) and on the pending and batch points: the base of ``NeiScorer`` (one target), ``ParegoScorer`` and
    ``NehviScorer``.  The winners of the family's pruning rule, counted over ``PRUNE_SAMPLES`` joint posterior
    samples, are every row once until the subclass prunes; every evaluation keeps at most ``MAX_PENDING`` - (its other
    conditioning points) of them and records how many it dropped in ``n_dropped``."""

    def __init__(self, gps, cfg: AcqConfig, baseline, prune: bool):
        self.gps, self.cfg, self.prune = list(gps), cfg, bool(prune)
        self.M = len(self.gps)
        self.device = self.gps[0].device
        self.baseline = np.asarray(baseline, dtype=np.float64).reshape(-1, self.gps[0].d)
        n = len(self.baseline)
        self.winners, self.counts = np.arange(n), np.ones(n, dtype=np.int64)
        self.n_dropped = 0

    def prune_samples(self, prune_seed: int, post=None):
        """The pruning draw: per target the float64 posterior mean of the baseline and the Cholesky factor of its
        covariance, and z (PRUNE_SAMPLES, M n), column block m for target m.  `post`: the (mean, covariance) pairs if
        the caller already has them."""
        from baybe_b200.multiobjective import _psd_cholesky

        n = len(self.baseline)
        if post is None:
            post = [_joint_posterior(gp, self.baseline)[:2] for gp in self.gps]
        Ls = [_psd_cholesky(0.5 * (cov + cov.T)) for _, cov in post]
        z = sobol_normal_samples(PRUNE_SAMPLES, self.M * n, prune_seed).numpy()
        return [mu for mu, _ in post], Ls, z

    # ---- candidate-independent set-up of one evaluation ----------------------------------------------------
    def kept_baseline(self, n_other: int) -> np.ndarray:
        """Indices of the baseline rows that condition an evaluation with `n_other` pending and batch points."""
        kept, self.n_dropped = capped_baseline(self.cfg.kind, self.winners, self.counts, len(self.baseline),
                                               self.prune, n_other)
        return kept

    def n_conditioning(self, n_other: int) -> int:
        return len(self.kept_baseline(n_other)) + n_other

    def n_sample_columns(self, n_other: int) -> int:
        """M(1 + |C|): per target block the conditioning points in the order of C, then the candidate."""
        return self.M * (1 + self.n_conditioning(n_other))

    def condition(self, pend: np.ndarray | None, batch: np.ndarray | None, z: np.ndarray):
        """C = [kept baseline; pending; batch] rows and, per target, L_C^-1 [M, |C|, |C|], w = (L_C^-T z_C)^T
        [M, S, |C|], the joint samples of C [S, |C|, M] and the (rows, beta) pair of C for ``cross_covariance``, all
        float64.  z: (S, M(1 + |C|)), column m(1 + |C|) + j = point j of target m."""
        d = self.gps[0].d
        pend = np.zeros((0, d)) if pend is None else np.asarray(pend, dtype=np.float64).reshape(-1, d)
        batch = np.zeros((0, d)) if batch is None else np.asarray(batch, dtype=np.float64).reshape(-1, d)
        rows = np.concatenate([self.baseline[self.kept_baseline(len(pend) + len(batch))], pend, batch])
        nc, M = len(rows), self.M
        if z.shape[1] != M * (nc + 1):
            raise ValueError(f"base samples must be (S, {M * (nc + 1)})")
        S = z.shape[0]
        linv, w, Y, conds = np.zeros((M, nc, nc)), np.zeros((M, S, nc)), np.zeros((S, nc, M)), []
        for m, gp in enumerate(self.gps if nc else ()):
            mu, L, linv[m], cond = condition_on(gp, rows)
            zc = z[:, m * (nc + 1): m * (nc + 1) + nc]
            Y[:, :, m] = mu[None, :] + zc @ L.T
            w[m] = zc @ linv[m]
            conds.append(cond)
        return rows, linv, w, Y, conds


class NeiScorer(BaselineScorer):
    """qNEI / qLogNEI over one single-task model with an affine objective o = a y + b (``cfg.obj_scale`` /
    ``cfg.obj_shift``).  `baseline`: the measured rows (raw comp-rep).  With `prune`, the baseline is pruned once,
    from ``PRUNE_SAMPLES`` joint posterior samples drawn with `prune_seed`, to the rows that are the arg-max of o in
    at least one sample."""

    def __init__(self, gp, cfg: AcqConfig, baseline, prune: bool = True, prune_seed: int = 0):
        if cfg.kind not in _lib.NEI_KINDS:
            raise ValueError(f"{cfg.kind} is not a noisy expected improvement")
        super().__init__([gp], cfg, baseline, prune)
        self.gp = gp
        n = len(self.baseline)
        if n == 0:
            raise ValueError("noisy expected improvement needs at least one measured row")
        if self.prune and n > 1:
            (mu,), (L,), z = self.prune_samples(prune_seed)
            self.winners, self.counts = prune_winners(cfg.obj_scale * (mu[None, :] + z @ L.T) + cfg.obj_shift)

    def conditioning(self, pend: np.ndarray | None, batch: np.ndarray | None, z: np.ndarray):
        """C = [kept baseline; pending; batch] rows, L_C^-1, w = (L_C^-T z_C)^T [S, |C|], the incumbents g [S] and the
        batch terms [S, Q] (None without batch points), all float64, and the (rows, beta) pair of C for
        ``cross_covariance``.  z: (S, 1 + |C|)."""
        rows, linv, w, Y, (cond,) = self.condition(pend, batch, z)
        nc, Q = len(rows), 0 if batch is None else len(batch)
        o = self.cfg.obj_scale * Y[:, :, 0] + self.cfg.obj_shift
        g = o[:, : nc - Q].max(axis=1)
        terms = None
        if Q:
            u = o[:, nc - Q:] - g[:, None]
            terms = _log_fatplus(u, self.cfg.tau_relu) if self.cfg.kind == "qLogNEI" else np.maximum(u, 0.0)
        return rows, linv[0], w[0], g, terms, cond

    def values(self, x, pend: np.ndarray | None, z: torch.Tensor, keep=None, index_offset: int = 0,
               want_scores: bool = True, batch: np.ndarray | None = None):
        """(scores or None, packed best key, report) for every row of x, conditional on the pending points and the
        other points of a q-batch (`batch`, whose per-sample terms join the candidate's); `report` is the identity."""
        z64 = torch.as_tensor(z, dtype=torch.float64).cpu().numpy()
        _, linv, w, g, terms, (px, beta) = self.conditioning(pend, batch, z64)
        dev, f32 = self.device, torch.float32
        mu, var, cross = self.gp.cross_covariance(self.gp.prepare(x), px, beta)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, f32)  # noqa: E731
        c = self.cfg
        scores, key = _nei_score(
            mu, var, cross.contiguous(), t(linv), t(w.T), t(z64), t(g), None if terms is None else t(terms), keep,
            c.kind == "qLogNEI", [c.obj_scale, c.obj_shift, c.tau_relu, c.tau_max], int(index_offset),
            bool(want_scores))
        return (scores if want_scores else None), key, (lambda v: v)

    def joint_value(self, rows, pend: np.ndarray | None, seed: int, n_samples: int) -> float:
        """Value of the q-batch `rows` given the pending points: the first row is the candidate, the others join
        the conditioning set and their per-sample terms join the candidate's."""
        rows = np.asarray(rows, dtype=np.float64).reshape(-1, self.gp.d)
        return float(self.scores(rows[:1], pend, seed, n_samples, batch=rows[1:])[0])


def build_nei_scorer(acqf, surrogate, searchspace, objective, measurements,
                     prune_seed: int = PRUNE_SEED) -> NeiScorer:
    """The reference's builder steps for the noisy-EI family (_builder.py:319-324) on the engine: check that the
    objective is affine in one modelled target, fit the surrogate, take the measured rows as baseline and prune it."""
    from baybe_b200.objectives import uses_objective_scorer
    from baybe_b200.searchspace import objective_affine

    name = type(acqf).__name__
    if uses_objective_scorer(objective):  # before the fit: a multi-model surrogate has no single device model
        raise NotImplementedError(
            f"'{name}' on the B200 engine needs an objective that is affine in one modelled target; "
            f"'{type(objective).__name__}' is not (a non-affine target transformation, or desirability computed on "
            "several models: use as_pre_transformation=True)")
    a, b, _ = objective_affine(objective)
    surrogate.fit(searchspace, objective, measurements)
    gp = surrogate.device_gp
    baseline = searchspace.transform(measurements, allow_extra=True).to_numpy(dtype=np.float64)
    cfg = AcqConfig(kind=acqf.abbreviation, obj_scale=a, obj_shift=b)
    return NeiScorer(gp, cfg, baseline, prune=acqf.prune_baseline, prune_seed=prune_seed)
