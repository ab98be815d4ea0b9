"""Pareto objectives on the engine: qExpectedHypervolumeImprovement and qLogExpectedHypervolumeImprovement over
discrete search spaces (``/root/reference/baybe/acquisition/acqfs.py:342-465``; context set up by
``acquisition/_builder.py:286-317``).

The host owns what does not depend on the candidate, in float64:
  * the reference point (``compute_ref_point`` of the oriented, fully measured targets, or the user's point);
  * the posterior-mean front F (the objective applied to every target's posterior mean at the training inputs);
  * an exact box decomposition of the region F does not dominate (``box_decomposition``), and with pending points
    one decomposition of F u P_s per base sample s together with the exact improvement of P_s over F.
``bb_hvi_score`` (csrc/mo.cu) evaluates the candidate-dependent improvement of every row on the device; the
sequential-greedy loop is ``baybe_b200.recommenders.greedy_select``.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.engine import AcqConfig
from baybe_b200.scoring import Scorer

class IncompleteMeasurementsError(Exception):
    """Same name/meaning as baybe.exceptions.IncompleteMeasurementsError."""


def _error(name: str) -> type[Exception]:
    """The reference's exception type of that name where baybe is importable (resolved at raise time: the package
    may be put on the path after this module was imported), else this package's twin."""
    try:
        import baybe.exceptions as bx

        return getattr(bx, name)
    except ImportError:  # pragma: no cover - baybe absent
        from baybe_b200 import acquisition

        return {"IncompleteMeasurementsError": IncompleteMeasurementsError,
                "IncompatibleAcquisitionFunctionError": acquisition.IncompatibleAcquisitionFunctionError}[name]


__all__ = ["compute_ref_point", "box_decomposition", "HviScorer", "build_hvi_scorer"]


def _hvi_score(*args):
    """``baybe_b200::hvi_score`` (engine.py); a module-level seam so that CPU tests can put a float64 stand-in here."""
    return torch.ops.baybe_b200.hvi_score(*args)


def compute_ref_point(array, maximize=None, factor: float = 0.1) -> np.ndarray:
    """``_ExpectedHypervolumeImprovement.compute_ref_point`` (acqfs.py:370-418): the worst point moved away from the
    best by `factor` times their difference, per target."""
    if np.ndim(array) != 2:
        raise ValueError("The specified data array must have exactly two dimensions.")
    if maximize is not None and np.ndim(maximize) != 1:
        raise ValueError("The specified Boolean array must have exactly one dimension.")
    array = np.asarray(array, dtype=np.float64)
    sign = np.where(np.ones(array.shape[1], bool) if maximize is None else np.asarray(maximize, bool), 1.0, -1.0)
    a = array * sign[None, :]
    lo, hi = a.min(axis=0), a.max(axis=0)
    return (lo - factor * (hi - lo)) * sign


def _pareto_points(Y: np.ndarray, ref: np.ndarray) -> np.ndarray:
    """Distinct non-dominated rows of Y that are strictly better than `ref` in every output (maximisation)."""
    Y = np.unique(Y[(Y > ref).all(axis=1)], axis=0)
    if len(Y) <= 1:
        return Y
    ge = (Y[:, None, :] >= Y[None, :, :]).all(-1)  # ge[i, j]: i weakly dominates j
    np.fill_diagonal(ge, False)
    return Y[~ge.any(axis=0)]


def _merge(lo: np.ndarray, hi: np.ndarray, dim: int) -> tuple[np.ndarray, np.ndarray]:
    """Join boxes that touch along `dim` and share every other bound (exact: the union is unchanged)."""
    if len(lo) <= 1:
        return lo, hi
    others = [j for j in range(lo.shape[1]) if j != dim]
    keys = [lo[:, dim]] + [hi[:, j] for j in others[::-1]] + [lo[:, j] for j in others[::-1]]
    order = np.lexsort(keys)
    lo, hi = lo[order], hi[order]
    same = (lo[1:, others] == lo[:-1, others]).all(1) & (hi[1:, others] == hi[:-1, others]).all(1)
    cont = np.concatenate([[False], same & (lo[1:, dim] == hi[:-1, dim])])
    start = np.flatnonzero(~cont)
    end = np.concatenate([start[1:], [len(lo)]]) - 1
    lo2, hi2 = lo[start].copy(), hi[start].copy()
    hi2[:, dim] = hi[end, dim]
    return lo2, hi2


# bound on (|F|+1)^(M-1) * |F|, the size of the grid's cover test: time and memory of one decomposition grow like
# |F|^M (on one CPU core about 20 ms at M = 3, |F| = 80 and 1.7 s at M = 4, |F| = 80)
MAX_GRID_WORK = 5e7


def box_decomposition(Y, ref) -> tuple[np.ndarray, np.ndarray, float]:
    """Exact decomposition of {y >= ref : y not dominated by Y} into disjoint boxes [lower, upper) (upper may be
    +inf), plus the hypervolume of Y relative to `ref`.  Maximisation; points not strictly better than `ref` in
    every output are dropped (botorch's partitionings do the same).

    Grid over the distinct coordinates of the front in the first M-1 outputs; every grid column is non-dominated
    above the highest last-output value among the points covering it, which gives one cell per column, and
    neighbouring cells are then joined along each output.  M = 2 yields the |F| + 1 staircase cells."""
    Y = np.asarray(Y, dtype=np.float64).reshape(-1, len(ref))
    ref = np.asarray(ref, dtype=np.float64)
    M = len(ref)
    F = _pareto_points(Y, ref)
    axes = [np.unique(np.concatenate([[ref[m]], F[:, m]])) for m in range(M - 1)]
    work = math.prod(len(a) for a in axes) * max(len(F), 1)
    if work > MAX_GRID_WORK:
        raise NotImplementedError(
            f"a front of {len(F)} points in {M} outputs needs a grid of {work:.2e} column-point tests "
            f"(limit {MAX_GRID_WORK:.0e}); reduce the number of targets or measurements")
    grids_lo = np.meshgrid(*axes, indexing="ij")
    grids_hi = np.meshgrid(*[np.append(a[1:], np.inf) for a in axes], indexing="ij")
    lo = np.stack([g.reshape(-1) for g in grids_lo], axis=1)
    hi = np.stack([g.reshape(-1) for g in grids_hi], axis=1)
    if len(F):
        cover = (F[None, :, : M - 1] >= hi[:, None, :]).all(-1)  # point f covers the whole column
        h = np.where(cover, F[None, :, M - 1], ref[M - 1]).max(axis=1)
    else:
        h = np.full(len(lo), ref[M - 1])
    finite = np.isfinite(hi).all(axis=1)
    hv = float((np.prod(hi[finite] - lo[finite], axis=1) * (h[finite] - ref[M - 1])).sum())
    lower = np.concatenate([lo, h[:, None]], axis=1)
    upper = np.concatenate([hi, np.full((len(lo), 1), np.inf)], axis=1)
    for dim in range(M - 2, -1, -1):
        lower, upper = _merge(lower, upper, dim)
    return lower, upper, hv


def hvi_hard(lower: np.ndarray, upper: np.ndarray, Y: np.ndarray) -> np.ndarray:
    """Hypervolume improvement of every row of Y (maximisation) over the cells: sum_c prod_m (min(y, u) - l)_+."""
    side = np.minimum(np.asarray(Y)[:, None, :], upper[None]) - lower[None]
    return np.clip(side, 0.0, None).prod(-1).sum(-1)


def _padded(decomps: list[tuple[np.ndarray, np.ndarray]], M: int):
    counts = np.array([len(lo) for lo, _ in decomps], dtype=np.int32)
    C = max(1, int(counts.max()))
    if C > _lib.HVI_MAX_CELLS:
        raise NotImplementedError(
            f"the box decomposition of the Pareto front has {C} cells, more than the {_lib.HVI_MAX_CELLS} "
            "bb_hvi_score supports; pass fewer targets or fewer measurements")
    lower = np.zeros((len(decomps), C, M), dtype=np.float32)
    upper = np.zeros((len(decomps), C, M), dtype=np.float32)
    for k, (lo, hi) in enumerate(decomps):
        lower[k, : len(lo)] = lo
        upper[k, : len(hi)] = hi
    return lower, upper, counts, C


class HviScorer(Scorer):
    """qEHVI / qLogEHVI over one model per target.  `scales`/`shifts` orient target m as o_m = a_m y_m + b_m;
    `front` holds the oriented posterior means at the training inputs; `ref_point` is in the oriented space."""

    def __init__(self, gps, cfg: AcqConfig, scales, shifts, ref_point, front):
        if cfg.kind not in _lib.HVI_KINDS:
            raise ValueError(f"{cfg.kind} is not a hypervolume acquisition function")
        self.gps, self.cfg = list(gps), cfg
        self.M = len(self.gps)
        if not 2 <= self.M <= _lib.HVI_MAX_TARGETS:
            raise _error("IncompatibleAcquisitionFunctionError")(
                f"{cfg.kind} on the B200 engine supports 2 to {_lib.HVI_MAX_TARGETS} targets (got {self.M}); "
                "above that the reference partitions approximately")
        self.a = np.asarray(scales, dtype=np.float64)
        self.b = np.asarray(shifts, dtype=np.float64)
        self.ref = np.asarray(ref_point, dtype=np.float64).reshape(self.M)
        self.front = np.asarray(front, dtype=np.float64).reshape(-1, self.M)
        self.lower, self.upper, self.hv_front = box_decomposition(self.front, self.ref)
        self.device = self.gps[0].device

    # ---- candidate-independent set-up of one evaluation ----------------------------------------------------
    def _pending_parts(self, pend: np.ndarray, z: torch.Tensor):
        """Per target: cross-covariance inputs, L_PP^-1 and L^-T z_P; per sample: decomposition of F u P_s and
        the exact improvement of P_s over F.  z: (S, M(1+P)) float64."""
        from baybe_b200.objectives import pending_conditioning

        S = z.shape[0]
        stats, linv, w, ys = pending_conditioning(self.gps, pend, z)
        ps = self.a * ys + self.b
        decomps, gain = [], np.zeros(S)
        for s in range(S):
            lo, hi, hv = box_decomposition(np.concatenate([self.front, ps[s]], axis=0), self.ref)
            decomps.append((lo, hi))
            gain[s] = hv - self.hv_front
        return stats, linv, w, decomps, float(gain.mean())

    def values(self, x, pend: np.ndarray | None, z: torch.Tensor, keep=None, index_offset: int = 0,
               want_scores: bool = True):
        """(improvement scores or None, packed best key, report) for every row of x: `report` maps a value of the
        kernel to the acquisition value of the batch [x; pending] (adds the pending points' own improvement)."""
        M = self.M
        P = 0 if pend is None else len(pend)
        z = torch.as_tensor(z, dtype=torch.float64).reshape(-1, M * (1 + P))
        xd = self.gps[0].prepare(x)
        if P == 0:
            post = [gp.posterior(xd) for gp in self.gps]
            cross = linv = w = None
            decomps, gain = [(self.lower, self.upper)], 0.0
        else:
            stats, linv_h, w_h, decomps, gain = self._pending_parts(np.asarray(pend, dtype=np.float64), z)
            post = [gp.cross_covariance(xd, px, beta) for gp, (px, beta) in zip(self.gps, stats)]
            cross = torch.stack([c for _, _, c in post]).contiguous()
            linv = torch.from_numpy(linv_h).to(self.device, torch.float32)
            w = torch.from_numpy(w_h).to(self.device, torch.float32)
        mu = torch.stack([p[0] for p in post]).contiguous()
        var = torch.stack([p[1] for p in post]).contiguous()
        lower, upper, counts, C = _padded(decomps, M)
        dev = self.device
        scores, key = _hvi_score(
            mu, var, cross, linv, w, z.to(dev, torch.float32).contiguous(), torch.from_numpy(lower).to(dev),
            torch.from_numpy(upper).to(dev), torch.from_numpy(counts).to(dev), keep, _lib.ACQ_KIND[self.cfg.kind],
            self.cfg.params(), [float(v) for v in self.a], [float(v) for v in self.b], int(index_offset),
            bool(want_scores))
        return (scores if want_scores else None), key, self._reporter(gain)

    def _reporter(self, gain: float):
        if gain <= 0.0:
            return lambda v: v
        if self.cfg.kind == "qEHVI":
            return lambda v: v + gain
        lg = math.log(gain)
        return lambda v: np.logaddexp(lg, v)

    def n_sample_columns(self, n_other: int) -> int:
        """M(1+P): column m(1+P)+j is pending point j of target m, the last column of each target block the
        candidate."""
        return self.M * (1 + n_other)


def _psd_cholesky(K: np.ndarray) -> np.ndarray:
    """Cholesky with the jitter ladder of linear_operator's psd_safe_cholesky (1e-8 * 10^i, float64)."""
    try:
        return np.linalg.cholesky(K)
    except np.linalg.LinAlgError:
        pass
    for i in range(6):
        try:
            return np.linalg.cholesky(K + 1e-8 * 10.0**i * np.eye(len(K)))
        except np.linalg.LinAlgError:
            continue
    raise FloatingPointError("pending-point covariance is not positive definite")


def target_orientations(objective) -> tuple[np.ndarray, np.ndarray]:
    """(a, b) of every target of a multi-target objective: o_m = a_m y_m + b_m (same rule as ``objective_affine``)."""
    from baybe_b200.searchspace import target_affine

    ab = np.array([target_affine(t) for t in objective.targets], dtype=np.float64)
    return ab[:, 0], ab[:, 1]


def build_hvi_scorer(acqf, gps, searchspace, objective, measurements) -> HviScorer:
    """The reference's builder steps for the hypervolume family (_builder.py:141-193, 286-317) on the engine:
    reference point, posterior-mean front and its partitioning.  `gps`: one DeviceGP per target, in target order."""
    alpha = getattr(acqf, "alpha", None)
    if alpha is not None and alpha > 0.0:
        raise _error("IncompatibleAcquisitionFunctionError")(
            f"{type(acqf).__name__}(alpha={alpha}): approximate partitioning is not supported by the B200 engine; "
            "use alpha=None or 0.0 (exact partitioning)")
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
    train_x = torch.from_numpy(searchspace.transform(measurements, allow_extra=True).to_numpy(dtype=np.float64))
    front = np.stack([gp.posterior(train_x)[0].double().cpu().numpy() for gp in gps], axis=1) * a + b
    cfg = AcqConfig(kind=acqf.abbreviation)
    return HviScorer(gps, cfg, a, b, ref, front)
