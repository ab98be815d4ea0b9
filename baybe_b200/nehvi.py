"""Pareto objectives with a noisy baseline: qNoisyExpectedHypervolumeImprovement over discrete search spaces
(``/root/reference/baybe/acquisition/acqfs.py:468-474``; reference point as for qEHVI, ``X_baseline`` = the measured
rows, ``acquisition/_builder.py:286-324``).

qEHVI partitions the posterior-mean front once.  qNEHVI samples the front instead: per base sample s it values the
candidate's improvement over F_s, the sampled outputs of the conditioning set, so every evaluation needs one exact
box decomposition per sample.  The host owns, in float64:
  * the reference point (``compute_ref_point`` of the oriented, fully measured targets, or the user's point);
  * the pruned baseline (botorch's ``prune_inferior_points_multi_objective``): the measured rows that are on the
    Pareto front (no deduplication) and strictly above the reference point in at least one of 2048 joint posterior
    samples, capped like ``baybe_b200.noisy`` at 31 conditioning points;
  * per target, the conditioning set C = [kept baseline; pending; other points of a q-batch] sampled jointly
    (``noisy.condition_on``).
The device builds the S decompositions of F_s u O_s (O_s: the samples of the other batch points) with
``bb_hvi_decompose`` (csrc/boxdec.cu) and scores every candidate conditionally on C against them with
``bb_hvi_score`` (kind qEHVI).  Pending points join the front, not the improvement (botorch's
``incremental_nehvi=True``); the other points of a q-batch add mean_s(hv(F_s u O_s) - hv(F_s)).
"""
from __future__ import annotations

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.engine import AcqConfig
from baybe_b200.noisy import PRUNE_SAMPLES, PRUNE_SEED, BaselineScorer

__all__ = ["pareto_mask", "NehviScorer", "build_nehvi_scorer"]

_PRUNE_CHUNK = 32  # pruning samples per dominance test: [chunk, n, n, M] booleans


def _hvi_score(*args):
    """``baybe_b200::hvi_score`` (engine.py); a module-level seam so that CPU tests can put a float64 stand-in here."""
    return torch.ops.baybe_b200.hvi_score(*args)


def _hvi_decompose(points: np.ndarray, ref: np.ndarray, device):
    """Exact box decompositions of the float32 values of the oriented points [S, n, M] (``baybe_b200::hvi_decompose``,
    cell stride ``HVI_MAX_CELLS``): (lower, upper, n_cells, hv).  A module-level seam like ``_hvi_score``: CPU tests
    put ``box_decomposition`` here."""
    pts = torch.from_numpy(np.ascontiguousarray(points, dtype=np.float32)).to(device)
    return torch.ops.baybe_b200.hvi_decompose(pts, None, [float(r) for r in ref], _lib.HVI_MAX_CELLS)


def pareto_mask(Y: np.ndarray, ref: np.ndarray) -> np.ndarray:
    """Y [..., n, M] -> [..., n]: the rows no other row dominates (>= everywhere, > somewhere; duplicates do not
    dominate each other) that are strictly above `ref` in every output (botorch ``is_non_dominated(deduplicate=False)``
    and the reference-point filter of ``prune_inferior_points_multi_objective``)."""
    ge = np.ones(Y.shape[:-1] + Y.shape[-2:-1], dtype=bool)  # [..., j, i]: row j >= row i in every output so far
    gt = np.zeros_like(ge)
    for m in range(Y.shape[-1]):  # one output at a time: no reduction over a short last axis
        a, b = Y[..., :, None, m], Y[..., None, :, m]
        ge &= a >= b
        gt |= a > b
    return ~(ge & gt).any(-2) & (Y > ref).all(-1)


class NehviScorer(BaselineScorer):
    """qNEHVI over one model per target.  `scales`/`shifts` orient target m as o_m = a_m y_m + b_m; `ref_point` is in
    the oriented space; `baseline`: the measured rows (raw comp-rep).  With `prune`, the baseline is pruned once, from
    ``PRUNE_SAMPLES`` joint posterior samples drawn with `prune_seed`, to the rows on the sampled Pareto front."""

    def __init__(self, gps, cfg: AcqConfig, scales, shifts, ref_point, baseline, prune: bool = True,
                 prune_seed: int = PRUNE_SEED):
        from baybe_b200.multiobjective import _error

        if cfg.kind not in _lib.NEHVI_KINDS:
            raise ValueError(f"{cfg.kind} is not a noisy hypervolume acquisition function")
        M = len(gps)
        if not 2 <= M <= _lib.HVI_MAX_TARGETS:
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"{cfg.kind} on the B200 engine supports 2 to {_lib.HVI_MAX_TARGETS} targets (got {M}); "
                "above that the reference partitions approximately")
        super().__init__(gps, cfg, baseline, prune)
        self.a = np.asarray(scales, dtype=np.float64).reshape(self.M)
        self.b = np.asarray(shifts, dtype=np.float64).reshape(self.M)
        self.ref = np.asarray(ref_point, dtype=np.float64).reshape(self.M)
        n = len(self.baseline)
        if self.prune and n > 0:
            mus, Ls, z = self.prune_samples(prune_seed)
            counts = np.zeros(n, dtype=np.int64)
            for s0 in range(0, PRUNE_SAMPLES, _PRUNE_CHUNK):
                zs = z[s0:s0 + _PRUNE_CHUNK]
                Y = np.stack([mus[m][None, :] + zs[:, m * n:(m + 1) * n] @ Ls[m].T for m in range(self.M)], -1)
                counts += pareto_mask(Y * self.a + self.b, self.ref).sum(0)
            self.winners = np.flatnonzero(counts)
            self.counts = counts[self.winners]

    def conditioning(self, pend: np.ndarray | None, batch: np.ndarray | None, z: np.ndarray):
        """C = [kept baseline; pending; batch] rows; per target L_C^-1 [M, |C|, |C|] and w = (L_C^-T z_C)^T
        [M, S, |C|], the oriented samples of C [S, |C|, M] and the (rows, beta) pair of C per target for
        ``cross_covariance``, all float64.  z: (S, M(1 + |C|)), column m(1 + |C|) + j = point j of target m."""
        rows, linv, w, Y, conds = self.condition(pend, batch, z)
        return rows, linv, w, (Y * self.a + self.b if len(rows) else Y), conds

    def _decompose(self, points: np.ndarray):
        lower, upper, n_cells, hv = _hvi_decompose(points, self.ref, self.device)
        worst = int(n_cells.max())
        if worst > _lib.HVI_MAX_CELLS:
            raise NotImplementedError(
                f"the box decomposition of the Pareto front has {worst} cells, more than the {_lib.HVI_MAX_CELLS} "
                "bb_hvi_score supports; pass fewer targets or fewer measurements")
        return lower, upper, n_cells, hv

    def values(self, x, pend: np.ndarray | None, z: torch.Tensor, keep=None, index_offset: int = 0,
               want_scores: bool = True, batch: np.ndarray | None = None):
        """(improvement scores or None, packed best key, report) for every row of x, conditional on the pending
        points and the other points of a q-batch (`batch`); `report` adds the batch points' own improvement
        mean_s(hv(F_s u O_s) - hv(F_s)) to a value of the kernel."""
        z64 = torch.as_tensor(z, dtype=torch.float64).cpu().numpy()
        rows, linv, w, o, conds = self.conditioning(pend, batch, z64)
        nc, Q = len(rows), 0 if batch is None else len(batch)
        dev, f32 = self.device, torch.float32
        xd = self.gps[0].prepare(x)
        gain = 0.0
        if nc == 0:  # nothing to condition on: one decomposition, of the empty front
            post = [gp.posterior(xd) for gp in self.gps]
            cross = linv_d = w_d = None
            lower, upper, n_cells, _ = self._decompose(np.zeros((1, 0, self.M)))
        else:
            post = [gp.cross_covariance(xd, px, beta) for gp, (px, beta) in zip(self.gps, conds)]
            cross = torch.stack([p[2] for p in post]).contiguous()
            linv_d = torch.from_numpy(linv).to(dev, f32)
            w_d = torch.from_numpy(w).to(dev, f32)
            lower, upper, n_cells, hv = self._decompose(o)
            if Q:
                hv_f = self._decompose(o[:, : nc - Q])[3] if nc > Q else torch.zeros_like(hv)
                gain = float((hv.double() - hv_f.double()).mean())
        mu = torch.stack([p[0] for p in post]).contiguous()
        var = torch.stack([p[1] for p in post]).contiguous()
        scores, key = _hvi_score(
            mu, var, cross, linv_d, w_d, torch.as_tensor(z64).to(dev, f32).contiguous(), lower, upper, n_cells,
            keep, _lib.ACQ_KIND["qEHVI"], AcqConfig(kind="qEHVI").params(), [float(v) for v in self.a],
            [float(v) for v in self.b], int(index_offset), bool(want_scores))
        return (scores if want_scores else None), key, ((lambda v: v + gain) if gain > 0.0 else (lambda v: v))

    def joint_value(self, rows, pend: np.ndarray | None, seed: int, n_samples: int) -> float:
        """Value of the q-batch `rows` given the pending points: the first row is the candidate, the others join
        the conditioning set and the sampled front's improvement."""
        rows = np.asarray(rows, dtype=np.float64).reshape(-1, self.gps[0].d)
        return float(self.scores(rows[:1], pend, seed, n_samples, batch=rows[1:])[0])


def build_nehvi_scorer(acqf, gps, searchspace, objective, measurements, prune_seed: int = PRUNE_SEED) -> NehviScorer:
    """The reference's builder steps for qNEHVI (_builder.py:286-324) on the engine: orient the targets, set the
    reference point as for qEHVI, take the measured rows as baseline and prune it.  `gps`: one DeviceGP per target,
    in target order (already fitted)."""
    from baybe_b200.multiobjective import _error, compute_ref_point, target_orientations

    names = [t.name for t in objective.targets]
    if not 2 <= len(names) <= _lib.HVI_MAX_TARGETS:
        raise _error("IncompatibleAcquisitionFunctionError")(
            f"{acqf.abbreviation} on the B200 engine supports 2 to {_lib.HVI_MAX_TARGETS} targets (got {len(names)})")
    a, b = target_orientations(objective)
    ref = acqf.reference_point
    if ref is None or isinstance(ref, float):
        complete = measurements[names].dropna()
        if complete.empty:
            raise _error("IncompleteMeasurementsError")(
                "For calculating a default reference point, at least one configuration must have a measured value "
                "for all targets. You can fix this by setting the 'reference_point' argument of "
                f"'{type(acqf).__name__}' explicitly.")
        oriented = complete.to_numpy(dtype=np.float64) * a[None, :] + b[None, :]
        ref = compute_ref_point(oriented, factor=0.1 if ref is None else ref)
    baseline = searchspace.transform(measurements, allow_extra=True).to_numpy(dtype=np.float64)
    return NehviScorer(gps, AcqConfig(kind=acqf.abbreviation), a, b, ref, baseline, prune=acqf.prune_baseline,
                       prune_seed=prune_seed)
