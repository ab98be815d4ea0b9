"""Pareto objectives by random Chebyshev scalarisation: qLogNParEGO over discrete search spaces
(``/root/reference/baybe/acquisition/acqfs.py:328-336``; ``X_baseline`` = the measured rows,
``acquisition/_builder.py:195-209, 319-334``).

Each scorer draws one set of simplex weights (botorch's ``sample_simplex``), normalises every oriented target by the
range of its posterior mean over the measured rows and scalarises by the augmented Chebyshev form
cheb(o) = min_m p_m + alpha sum_m p_m, p_m = lambda_m (o_m - lo_m) / (hi_m - lo_m); the host folds orientation,
normalisation and weight into one affine map per target, p_m = W_m y_m + V_m.  The value is a qLogNEI of cheb over a
pruned baseline, set up as in ``baybe_b200.noisy`` in float64 on the host:
  * the pruned baseline: the measured rows that are the arg-max of cheb in at least one of 2048 joint posterior
    samples (one ``bb_joint_posterior`` per target model);
  * per target, the conditioning set C = [kept baseline; pending; other points of a q-batch] sampled jointly, the
    per-sample incumbent g_s (the hard maximum of cheb over baseline and pending points) and the per-sample terms of
    the other batch points.
``bb_parego_score`` (csrc/parego.cu) samples every candidate conditionally on C per target and reduces over the
samples on the device.  Unlike qEHVI its cost is linear in the number of targets, so it serves up to 8.
"""
from __future__ import annotations

import numpy as np
import torch

from baybe_b200 import _lib, noisy
from baybe_b200.engine import AcqConfig, sobol_normal_samples
from baybe_b200.noisy import PRUNE_SAMPLES, PRUNE_SEED, _log_fatplus, capped_baseline, condition_on, prune_winners

__all__ = ["CHEBYSHEV_ALPHA", "sample_simplex", "chebyshev", "ParegoScorer", "build_parego_scorer"]

CHEBYSHEV_ALPHA = 0.05  # botorch get_chebyshev_scalarization's alpha


def _parego_score(*args):
    """``baybe_b200::parego_score`` (engine.py); a module-level seam so that CPU tests can put a float64 stand-in
    here."""
    return torch.ops.baybe_b200.parego_score(*args)


def sample_simplex(M: int) -> np.ndarray:
    """One point drawn uniformly from the (M-1)-simplex as botorch's ``sample_simplex(M, n=1)`` draws it: the gaps
    of [0, sort(u), 1] for u = ``torch.rand(1, M - 1, dtype=float64)`` from torch's global RNG."""
    u = torch.rand(1, M - 1, dtype=torch.float64)
    s = torch.cat([torch.zeros(1, 1, dtype=torch.float64), torch.sort(u, dim=-1).values,
                   torch.ones(1, 1, dtype=torch.float64)], dim=-1)
    return (s[0, 1:] - s[0, :-1]).numpy()


def chebyshev(p: np.ndarray, alpha: float = CHEBYSHEV_ALPHA) -> np.ndarray:
    """Augmented Chebyshev scalarisation of the weighted normalised targets p [..., M]."""
    return p.min(axis=-1) + alpha * p.sum(axis=-1)


class ParegoScorer:
    """qLogNParEGO over one model per target; the interface of ``NeiScorer`` (``values``, ``round_best``, ``scores``,
    ``base_samples``, ``joint_value``, ``n_dropped``).  `scales`/`shifts` orient target m as o_m = a_m y_m + b_m;
    `baseline`: the measured rows (raw comp-rep); `weights`: the simplex weights lambda.  The normalisation bounds
    lo_m, hi_m are the extremes of the oriented float64 posterior mean over every measured row; a range that is not
    positive counts as 1 (botorch would divide by zero).  With `prune`, the baseline is pruned once on the
    scalarised objective, from ``PRUNE_SAMPLES`` joint posterior samples drawn with `prune_seed`."""

    def __init__(self, gps, cfg: AcqConfig, scales, shifts, baseline, weights, prune: bool = True,
                 prune_seed: int = PRUNE_SEED):
        if cfg.kind not in _lib.PAREGO_KINDS:
            raise ValueError(f"{cfg.kind} is not a ParEGO acquisition function")
        self.gps, self.cfg, self.prune = list(gps), cfg, bool(prune)
        self.M = len(self.gps)
        if not 2 <= self.M <= _lib.PAREGO_MAX_TARGETS:
            from baybe_b200.multiobjective import _error

            raise _error("IncompatibleAcquisitionFunctionError")(
                f"{cfg.kind} on the B200 engine supports 2 to {_lib.PAREGO_MAX_TARGETS} targets (got {self.M})")
        self.device = self.gps[0].device
        self.a = np.asarray(scales, dtype=np.float64).reshape(self.M)
        self.b = np.asarray(shifts, dtype=np.float64).reshape(self.M)
        self.weights = np.asarray(weights, dtype=np.float64).reshape(self.M)
        self.alpha = CHEBYSHEV_ALPHA
        self.baseline = np.asarray(baseline, dtype=np.float64).reshape(-1, self.gps[0].d)
        n = len(self.baseline)
        if n == 0:
            raise ValueError("qLogNParEGO needs at least one measured row")
        post = [noisy._joint_posterior(gp, self.baseline)[:2] for gp in self.gps]
        o = np.stack([mu for mu, _ in post], axis=1) * self.a + self.b  # oriented posterior means [n, M]
        lo, hi = o.min(axis=0), o.max(axis=0)
        rng = np.where(hi - lo > 0.0, hi - lo, 1.0)
        self.W = self.weights * self.a / rng  # p_m = W_m y_m + V_m
        self.V = self.weights * (self.b - lo) / rng
        self.winners, self.counts = np.arange(n), np.ones(n, dtype=np.int64)
        if self.prune and n > 1:
            from baybe_b200.multiobjective import _psd_cholesky

            z = sobol_normal_samples(PRUNE_SAMPLES, self.M * n, prune_seed).numpy()
            Y = np.stack([mu[None, :] + z[:, m * n:(m + 1) * n] @ _psd_cholesky(0.5 * (cov + cov.T)).T
                          for m, (mu, cov) in enumerate(post)], axis=-1)  # [samples, n, M]
            self.winners, self.counts = prune_winners(chebyshev(self.W * Y + self.V, self.alpha))
        self.n_dropped = 0

    # ---- candidate-independent set-up of one evaluation ----------------------------------------------------
    def kept_baseline(self, n_other: int) -> np.ndarray:
        """Indices of the baseline rows that condition an evaluation with `n_other` pending and batch points."""
        kept, self.n_dropped = capped_baseline(self.cfg.kind, self.winners, self.counts, len(self.baseline),
                                               self.prune, n_other)
        return kept

    def n_conditioning(self, n_other: int) -> int:
        return len(self.kept_baseline(n_other)) + n_other

    def conditioning(self, pend: np.ndarray | None, batch: np.ndarray | None, z: np.ndarray):
        """C = [kept baseline; pending; batch] rows; per target L_C^-1 [M, |C|, |C|], w = (L_C^-T z_C)^T [M, S, |C|]
        and the (rows, beta) pair of C for ``cross_covariance``; the incumbents g [S] and the batch terms [S, Q]
        (None without batch points), all float64.  z: (S, M(1 + |C|)), column m(1 + |C|) + j = point j of target m."""
        d = self.gps[0].d
        pend = np.zeros((0, d)) if pend is None else np.asarray(pend, dtype=np.float64).reshape(-1, d)
        batch = np.zeros((0, d)) if batch is None else np.asarray(batch, dtype=np.float64).reshape(-1, d)
        rows = np.concatenate([self.baseline[self.kept_baseline(len(pend) + len(batch))], pend, batch])
        nc, Q, M = len(rows), len(batch), self.M
        if z.shape[1] != M * (nc + 1):
            raise ValueError(f"base samples must be (S, {M * (nc + 1)})")
        S = z.shape[0]
        linv, w, Y, conds = np.zeros((M, nc, nc)), np.zeros((M, S, nc)), np.zeros((S, nc, M)), []
        for m, gp in enumerate(self.gps):
            mu, L, linv[m], cond = condition_on(gp, rows)
            zc = z[:, m * (nc + 1): m * (nc + 1) + nc]
            Y[:, :, m] = mu[None, :] + zc @ L.T
            w[m] = zc @ linv[m]
            conds.append(cond)
        cheb = chebyshev(self.W * Y + self.V, self.alpha)  # [S, |C|]
        g = cheb[:, : nc - Q].max(axis=1)
        terms = _log_fatplus(cheb[:, nc - Q:] - g[:, None], self.cfg.tau_relu) if Q else None
        return rows, linv, w, g, terms, conds

    def values(self, x, pend: np.ndarray | None, z: torch.Tensor, keep=None, index_offset: int = 0,
               want_scores: bool = True, batch: np.ndarray | None = None):
        """(scores or None, packed best key, report) for every row of x, conditional on the pending points and the
        other points of a q-batch (`batch`, whose per-sample terms join the candidate's); `report` is the identity."""
        z64 = torch.as_tensor(z, dtype=torch.float64).cpu().numpy()
        _, linv, w, g, terms, conds = self.conditioning(pend, batch, z64)
        dev, f32 = self.device, torch.float32
        xd = self.gps[0].prepare(x)
        post = [gp.cross_covariance(xd, px, beta) for gp, (px, beta) in zip(self.gps, conds)]
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, f32)  # noqa: E731
        c = self.cfg
        scores, key = _parego_score(
            torch.stack([p[0] for p in post]).contiguous(), torch.stack([p[1] for p in post]).contiguous(),
            torch.stack([p[2] for p in post]).contiguous(), t(linv), t(w.transpose(0, 2, 1)), t(z64), t(g),
            None if terms is None else t(terms), keep, [float(v) for v in self.W], [float(v) for v in self.V],
            [self.alpha, c.tau_relu, c.tau_max], int(index_offset), bool(want_scores))
        return (scores if want_scores else None), key, (lambda v: v)

    # ---- the interfaces the recommenders use -------------------------------------------------------------------
    def base_samples(self, n_samples: int, n_pending: int, seed: int) -> torch.Tensor:
        """Scrambled Sobol normals of dimension M(1 + |C|): per target block the conditioning points in the order of
        C, then the candidate."""
        return sobol_normal_samples(n_samples, self.M * (1 + self.n_conditioning(n_pending)), seed)

    def round_best(self, x, pend: np.ndarray, keep, index_offset: int, seed: int, n_samples: int):
        """One sequential-greedy round: (packed best key, report) -- see ``greedy_select``."""
        P = len(pend)
        _, key, report = self.values(x, pend if P else None, self.base_samples(n_samples, P, seed), keep,
                                     index_offset, want_scores=False)
        return key, report

    def scores(self, x, pend: np.ndarray | None, seed: int, n_samples: int, batch: np.ndarray | None = None):
        """Acquisition value of every row given the pending points (and the other points of its q-batch), float64."""
        n_other = (0 if pend is None else len(pend)) + (0 if batch is None else len(batch))
        z = self.base_samples(n_samples, n_other, seed)
        s, _, _ = self.values(x, pend if pend is not None and len(pend) else None, z,
                              batch=batch if batch is not None and len(batch) else None)
        return s.double().cpu().numpy()

    def joint_value(self, rows, pend: np.ndarray | None, seed: int, n_samples: int) -> float:
        """Value of the q-batch `rows` given the pending points: the first row is the candidate, the others join
        the conditioning set and their per-sample terms join the candidate's."""
        rows = np.asarray(rows, dtype=np.float64).reshape(-1, self.gps[0].d)
        return float(self.scores(rows[:1], pend, seed, n_samples, batch=rows[1:])[0])


def build_parego_scorer(acqf, gps, searchspace, objective, measurements, prune_seed: int = PRUNE_SEED) -> ParegoScorer:
    """The reference's builder steps for qLogNParEGO (_builder.py:195-209, 319-334) on the engine: orient the targets,
    draw the simplex weights from torch's global RNG (once per construction, before the sampler seed), take the
    measured rows as baseline and prune it.  `gps`: one DeviceGP per target, in target order (already fitted)."""
    from baybe_b200.multiobjective import target_orientations

    a, b = target_orientations(objective)
    baseline = searchspace.transform(measurements, allow_extra=True).to_numpy(dtype=np.float64)
    weights = sample_simplex(len(gps))
    return ParegoScorer(gps, AcqConfig(kind=acqf.abbreviation), a, b, baseline, weights,
                        prune=acqf.prune_baseline, prune_seed=prune_seed)
