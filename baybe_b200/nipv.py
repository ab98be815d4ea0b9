"""Global active learning on discrete search spaces: qNegIntegratedPosteriorVariance
(``/root/reference/baybe/acquisition/acqfs.py:28-138``).

The value of a candidate x given the conditioning set C (pending points and the other points of a q-batch, observed
with noise) is the negative posterior variance averaged over fixed integration points m:

    qNIPV(x | C) = -(1/M) sum_m Var[f(m) | D, y(x), y(C)] = -(1/M) [ sum_m k_C(m,m) - IVR(x) ]

with k_C the posterior covariance given D and y(C), IVR(x) = sum_m k_C(m,x)^2 / (k_C(x,x) + sigma_n^2(x)).  The
variance does not depend on the fantasised values, so no samples are involved.  The host conditions on C in float64
(``bb_joint_posterior``, plus the noise, then the Cholesky factor), runs ``bb_posterior`` with C as its pending points
for the candidates and the integration points, and sums k_C(m,m) in float64; ``bb_nipv_score`` (csrc/nipv.cu) ranks
the candidates by IVR.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.engine import AcqConfig
from baybe_b200.noisy import _joint_posterior
from baybe_b200.scoring import Scorer

__all__ = ["NipvScorer", "sample_integration_points"]


def _nipv_score(*args):
    """``baybe_b200::nipv_score`` (engine.py); a module-level seam so that CPU tests can put a float64 stand-in here."""
    return torch.ops.baybe_b200.nipv_score(*args)


def sample_integration_points(comp_rep, n_points: int | None, fraction: float | None, method: str = "Random"):
    """Integration rows drawn from the full discrete comp-rep as the reference's ``get_integration_points`` and
    ``sample_numerical_df`` draw them: n = `n_points` or ceil(`fraction` * rows); whole copies of the frame for every
    full multiple of its length, then the remainder sampled with pandas' ``sample`` on the global NumPy RNG."""
    if method != "Random":
        raise NotImplementedError(
            f"sampling_method={method!r}: farthest-point sampling builds an N x N distance matrix on the host; use "
            "the BayBE spec's get_integration_points (the plugin does) or sampling_method='Random'")
    n = n_points or math.ceil(fraction * len(comp_rep))
    n_trivial, n_sampled = divmod(n, len(comp_rep))
    ilocs = list(range(len(comp_rep))) * n_trivial
    if n_sampled > 0:
        ilocs += comp_rep.reset_index(drop=True).sample(n_sampled).index.tolist()
    return comp_rep.iloc[ilocs]


def _tasks(rows: np.ndarray, gp) -> np.ndarray:
    if gp.task_col is None:
        return np.zeros(len(rows), dtype=np.int64)
    return np.clip(np.rint(rows[:, gp.task_col]).astype(np.int64), 0, gp.n_tasks - 1)


class NipvScorer(Scorer):
    """qNIPV over one model; `integration`: the integration rows (raw comp-rep), sent to the device once."""

    def __init__(self, gp, cfg: AcqConfig, integration):
        from baybe_b200.engine import nipv_model_terms

        if cfg.kind not in _lib.NIPV_KINDS:
            raise ValueError(f"{cfg.kind} is not an integrated posterior variance")
        if gp.n > _lib.NIPV_MAX_TRAIN:
            raise NotImplementedError(
                f"qNIPV on the B200 engine supports models of at most {_lib.NIPV_MAX_TRAIN} training points "
                f"(got {gp.n})")
        if getattr(gp.model, "wide", 0):
            raise NotImplementedError("qNIPV on the B200 engine does not support wide-feature models")
        self.gp, self.cfg, self.device = gp, cfg, gp.device
        xm = np.asarray(integration, dtype=np.float64).reshape(-1, gp.d)
        if len(xm) == 0:
            raise ValueError("qNIPV needs at least one integration point")
        self.M = len(xm)
        self.xm = torch.from_numpy(np.ascontiguousarray(xm, dtype=np.float32)).to(self.device)
        noise, _ = nipv_model_terms(gp)
        self.noise = np.asarray(noise, dtype=np.float64)
        self.y_var = float(gp.model.y_std) ** 2

    def n_sample_columns(self, n_other: int) -> None:
        return None

    def conditioning(self, pend: np.ndarray | None, batch: np.ndarray | None):
        """C = [pending; batch] rows, L_C^-1 of K_D(C,C) + diag sigma_n^2(C) (original units, float64) and the (rows,
        beta) pair of C for ``cross_covariance``; empty C: (rows, None, None)."""
        d = self.gp.d
        parts = [np.asarray(p, dtype=np.float64).reshape(-1, d) for p in (pend, batch) if p is not None]
        rows = np.concatenate(parts) if parts else np.zeros((0, d))
        if len(rows) > _lib.MAX_PENDING:
            raise NotImplementedError(
                f"qNIPV conditions on at most {_lib.MAX_PENDING} pending and batch points (got {len(rows)})")
        if len(rows) == 0:
            return rows, None, None
        _, cov, cond = _joint_posterior(self.gp, rows, with_beta=True)
        K = 0.5 * (cov + cov.T) + np.diag(self.noise[_tasks(rows, self.gp)] * self.y_var)
        return rows, np.linalg.inv(np.linalg.cholesky(K)), cond

    def values(self, x, pend: np.ndarray | None, z=None, keep=None, index_offset: int = 0,
               want_scores: bool = True, batch: np.ndarray | None = None):
        """(IVR scores or None, packed best key, report) for every row of x given the pending points and the other
        points of a q-batch; `report` maps IVR to qNIPV (original units)."""
        rows, linv, cond = self.conditioning(pend, batch)
        gp, dev = self.gp, self.device
        xd = gp.prepare(x)
        if xd.dtype != torch.float32 or not xd.is_contiguous() or xd.stride(-1) != 1:
            xd = xd.to(torch.float32).contiguous()
        if linv is None:
            _, var = gp.posterior(xd)
            _, var_m = gp.posterior(self.xm)
            cross = cross_m = linv_d = None
            kc_mm = float(var_m.double().sum())
        else:
            px, beta = cond
            _, var, cross = gp.cross_covariance(xd, px, beta)
            _, var_m, cross_m = gp.cross_covariance(self.xm, px, beta)
            linv_d = torch.from_numpy(linv).to(dev)
            kc_mm = float((var_m.double() - ((cross_m.double() @ linv_d.T) ** 2).sum(1)).sum())
        scores, key = _nipv_score(xd, self.xm, var, cross, cross_m, linv_d, keep, gp.handle,
                                  int(index_offset), bool(want_scores))
        M = self.M
        return (scores if want_scores else None), key, (lambda v: (np.asarray(v, dtype=np.float64) - kc_mm) / M)
