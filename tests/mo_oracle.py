"""Float64 oracle of the hypervolume acquisition functions (qEHVI / qLogEHVI, baybe/acquisition/acqfs.py:421-451,
context from acquisition/_builder.py:286-317) -- test infrastructure only.

  * ``hv``: exact hypervolume by brute force over the full coordinate grid (independent of the product's
    box decomposition);
  * ``cell_values``: hard / smoothed improvement of samples over given cells (the kernel's definition);
  * ``ehvi``: the engine's evaluation form -- conditional candidate samples, one decomposition of F u P_s per
    sample, plus the exact improvement of the pending points;
  * ``inclusion_exclusion``: the literal q-batch form (joint samples of [pending; x], inclusion-exclusion over the
    subsets of the batch; botorch's smoothed version for qLogEHVI), the independent check of the incremental form.
The cells come from ``baybe_b200.multiobjective.box_decomposition``: the smoothed value depends on the partitioning,
so the kernel and the oracle must share it; the partitioning itself is checked against ``hv`` in tests/test_mo.py.
"""
from __future__ import annotations

import itertools
import math

import numpy as np
import torch

import oracle
from oracle.reference_path import _log_fatplus
from baybe_b200.multiobjective import box_decomposition

TAU_RELU, TAU_MAX = 1e-6, 1e-2


def hv(Y, ref) -> float:
    """Hypervolume of the region dominated by Y above ref (maximisation), summed over the full coordinate grid."""
    Y = np.asarray(Y, dtype=np.float64).reshape(-1, len(ref))
    Y = Y[(Y > ref).all(1)]
    if len(Y) == 0:
        return 0.0
    axes = [np.unique(np.concatenate([[ref[m]], Y[:, m]])) for m in range(len(ref))]
    lo = np.stack(np.meshgrid(*[a[:-1] for a in axes], indexing="ij"), -1).reshape(-1, len(ref))
    hi = np.stack(np.meshgrid(*[a[1:] for a in axes], indexing="ij"), -1).reshape(-1, len(ref))
    dom = (Y[None, :, :] >= hi[:, None, :]).all(-1).any(-1)
    return float(np.prod(hi[dom] - lo[dom], axis=1).sum())


def _fatmin(a: torch.Tensor, b: torch.Tensor, tau: float) -> torch.Tensor:
    """botorch fatminimum: -fatmax(-a, -b) with alpha = 2; exactly a where b = +inf."""
    m = torch.minimum(a, b)
    d = torch.where(torch.isinf(b), torch.full_like(a, math.inf), (a - b).abs())
    return m - tau * torch.log1p((1.0 + d / (2.0 * tau)) ** -2)


def cell_values(Y: torch.Tensor, lower, upper, log: bool, tau_relu=TAU_RELU, tau_max=TAU_MAX) -> torch.Tensor:
    """Y [..., M] -> hard HVI sum_c prod_m (min(y, u) - l)_+  or  log sum_c prod_m fatplus(fatmin(y, u) - l)."""
    lo = torch.as_tensor(lower, dtype=torch.float64)
    up = torch.as_tensor(upper, dtype=torch.float64)
    y = Y[..., None, :]
    if not log:
        return (torch.minimum(y, up) - lo).clamp_min(0.0).prod(-1).sum(-1)
    if lo.shape[0] == 0:
        return torch.full(Y.shape[:-1], -math.inf, dtype=torch.float64)
    return torch.logsumexp(_log_fatplus(_fatmin(y, up, tau_max) - lo, tau_relu).sum(-1), dim=-1)


def ehvi(oms, kind: str, a, b, ref, front, X, pend, z, chunk: int = 256) -> torch.Tensor:
    """Engine form of qEHVI / qLogEHVI of [x; pending] for every row of X (float64, CPU).
    a, b: orientation per target; ref: reference point; front: oriented posterior-mean front; z: (S, M(1+P))."""
    M = len(oms)
    P = 0 if pend is None else len(pend)
    Q = P + 1
    z = torch.as_tensor(z, dtype=torch.float64).reshape(-1, M * Q)
    S = z.shape[0]
    log = kind == "qLogEHVI"
    a = torch.as_tensor(np.asarray(a, dtype=np.float64))
    b = torch.as_tensor(np.asarray(b, dtype=np.float64))
    X = np.asarray(X, dtype=np.float64)
    lo0, up0, hv0 = box_decomposition(front, ref)
    if P == 0:
        cells = [(lo0, up0)]
        gain = 0.0
    else:
        pm = [oracle.posterior_joint(om, pend) for om in oms]
        Ls = [torch.linalg.cholesky(c) for _, c in pm]
        ps = torch.stack([a[m] * (pm[m][0][None, :] + z[:, m * Q: m * Q + P] @ Ls[m].T) + b[m] for m in range(M)], -1)
        cells, gains = [], []
        for s in range(S):
            lo, up, hvs = box_decomposition(np.concatenate([front, ps[s].numpy()]), ref)
            cells.append((lo, up))
            gains.append(hvs - hv0)
        gain = float(np.mean(gains))
    out = torch.empty(len(X), dtype=torch.float64)
    for c0 in range(0, len(X), chunk):
        xs = X[c0: c0 + chunk]
        Y = torch.empty(S, len(xs), M, dtype=torch.float64)
        for m, om in enumerate(oms):
            mu, var = oracle.posterior(om, xs)
            zx = z[:, m * Q + P]
            if P == 0:
                Y[:, :, m] = mu[None, :] + var.sqrt()[None, :] * zx[:, None]
            else:
                sub = np.concatenate([pend, xs])
                mj, cj = oracle.posterior_joint(om, sub)
                cxp = cj[P:, :P]  # (n, P)
                r = torch.linalg.solve_triangular(Ls[m], cxp.T, upper=False).T  # Sigma_xP L^-T
                sd = (var - (r * r).sum(1)).clamp_min(0.0).sqrt()
                Y[:, :, m] = mu[None, :] + z[:, m * Q: m * Q + P] @ r.T + sd[None, :] * zx[:, None]
        Y = a * Y + b
        if P == 0:
            v = cell_values(Y, *cells[0], log=log)  # (S, n)
        else:
            v = torch.stack([cell_values(Y[s], *cells[s], log=log) for s in range(S)])
        val = (torch.logsumexp(v, 0) - math.log(S)) if log else v.mean(0)
        if gain > 0:
            val = torch.logaddexp(val, torch.tensor(math.log(gain), dtype=torch.float64)) if log else val + gain
        out[c0: c0 + chunk] = val
    return out


def inclusion_exclusion(oms, kind: str, a, b, ref, front, x_row, pend, z, tau_relu=TAU_RELU,
                        tau_max=TAU_MAX) -> float:
    """Literal q-batch value of [pending; x] (q + p <= 4): joint samples in the order [pending; x], inclusion-
    exclusion over the subsets of the batch against the cells of F (botorch qEHVI / qLogEHVI)."""
    M = len(oms)
    P = 0 if pend is None else len(pend)
    Q = P + 1
    z = torch.as_tensor(z, dtype=torch.float64).reshape(-1, M * Q)
    rows = np.asarray(x_row, dtype=np.float64).reshape(1, -1) if P == 0 else \
        np.concatenate([pend, np.asarray(x_row, dtype=np.float64).reshape(1, -1)])
    lo, up, _ = box_decomposition(front, ref)
    lo_t, up_t = torch.as_tensor(lo), torch.as_tensor(up)
    Y = []
    for m, om in enumerate(oms):
        mu, cov = oracle.posterior_joint(om, rows)
        L = torch.linalg.cholesky(cov)
        Y.append(float(a[m]) * (mu[None, :] + z[:, m * Q:(m + 1) * Q] @ L.T) + float(b[m]))
    Y = torch.stack(Y, -1)  # (S, Q, M)
    log = kind == "qLogEHVI"
    odd, even = [], []
    for k in range(1, Q + 1):
        for J in itertools.combinations(range(Q), k):
            sub = Y[:, list(J), :]  # (S, k, M)
            if log:
                from oracle.reference_path import _fatmax

                corner = -_fatmax(-sub, tau_max, dim=1) if k > 1 else sub[:, 0, :]
                t = _log_fatplus(_fatmin(corner[:, None, :], up_t, tau_max) - lo_t, tau_relu).sum(-1)
                val = torch.logsumexp(t, -1)
            else:
                corner = sub.amin(1)
                val = (torch.minimum(corner[:, None, :], up_t) - lo_t).clamp_min(0.0).prod(-1).sum(-1)
            (odd if k % 2 else even).append(val)
    S = Y.shape[0]
    if not log:
        return float((sum(odd) - (sum(even) if even else 0.0)).mean())
    lo_ = torch.logsumexp(torch.stack(odd), 0)
    if even:
        le = torch.logsumexp(torch.stack(even), 0)
        per = lo_ + torch.log1p(-torch.exp((le - lo_).clamp_max(0.0)))
    else:
        per = lo_
    return float(torch.logsumexp(per, 0) - math.log(S))
