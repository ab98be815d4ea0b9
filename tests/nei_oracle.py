"""Float64 definitions of the noisy expected improvement (test infrastructure): the arithmetic of csrc/nei.cu
(``nei_values_f64`` / ``nei_score_f64``, a stand-in for ``baybe_b200::nei_score``), the value from the full joint
Cholesky of [C; x] (``nei_full_joint``), and an engine stand-in whose joint posterior is the oracle's."""
from __future__ import annotations

import math

import numpy as np
import torch

import oracle
from oracle.reference_path import _fatmax, _log_fatplus
from tests.helpers import OracleBackedGP

F64 = torch.float64


def _reduce(t: torch.Tensor, terms, log_nei: bool, tau_max: float) -> torch.Tensor:
    """t [N, S] candidate terms, terms [S, Q] or None -> value per candidate."""
    S = t.shape[1]
    if terms is not None and terms.shape[1] > 0:
        tt = torch.as_tensor(terms, dtype=F64).to(t.device)
        allt = torch.cat([t[:, :, None], tt[None].expand(t.shape[0], -1, -1)], -1)
        t = _fatmax(allt, tau_max, dim=-1) if log_nei else allt.amax(-1)
    if log_nei:
        return torch.logsumexp(t, 1) - math.log(S)
    return t.mean(1)


def _terms(u: torch.Tensor, log_nei: bool, tau_relu: float) -> torch.Tensor:
    return _log_fatplus(u, tau_relu) if log_nei else u.clamp_min(0.0)


def nei_values_f64(mu, var, cross, linv, w_cs, zx, g, terms, log_nei: bool, a: float, b: float, tau_relu: float,
                   tau_max: float) -> torch.Tensor:
    """The definition of bb_nei_score in float64: mu/var [N], cross [N, C] or None, linv [C, C], w_cs [C, S]
    (sample-minor), zx [S] (the candidate's base samples), g [S], terms [S, Q] or None."""
    dev = mu.device if torch.is_tensor(mu) else torch.device("cpu")
    t64 = lambda v: (v.to(dev, F64) if torch.is_tensor(v)  # noqa: E731
                     else torch.as_tensor(np.asarray(v), dtype=F64, device=dev))
    mu, var, zx, g = t64(mu), t64(var), t64(zx), t64(g)
    if cross is not None and cross.shape[1] > 0:
        c = t64(cross)
        r = c @ t64(linv).T
        r2, dm = (r * r).sum(1), c @ t64(w_cs)
    else:
        r2, dm = torch.zeros_like(mu), torch.zeros(len(mu), len(zx), dtype=F64, device=dev)
    sd = (var - r2).clamp_min(0.0).sqrt()
    o = a * (mu[:, None] + dm + sd[:, None] * zx[None, :]) + b
    return _reduce(_terms(o - g[None, :], log_nei, tau_relu), terms, log_nei, tau_max)


def nei_score_f64(mu, var, cross, linv, w, z, g, batch_terms, keep, log_nei, params, index_offset, want_scores):
    """Float64 stand-in of ``baybe_b200::nei_score`` (same arguments)."""
    from baybe_b200.engine import pack_best

    cpu = lambda v: None if v is None else v.detach().double().cpu()  # noqa: E731
    a, b, tau_relu, tau_max = params
    zc = cpu(z)
    val = nei_values_f64(cpu(mu), cpu(var), cpu(cross), cpu(linv), cpu(w), zc[:, -1], cpu(g), cpu(batch_terms),
                         bool(log_nei), a, b, tau_relu, tau_max)
    s32 = val.float()
    best = -(1 << 63)
    for i in range(len(s32)):
        if (keep is None or int(keep[i]) != 0) and not math.isnan(float(s32[i])):
            best = max(best, pack_best(float(s32[i]), i + int(index_offset)))
    return (s32 if want_scores else None), torch.tensor([best], dtype=torch.int64)


def nei_full_joint(om, rows: np.ndarray, n_incumbent: int, x: np.ndarray, z: np.ndarray, log_nei: bool, a: float,
                   b: float, tau_relu: float, tau_max: float) -> torch.Tensor:
    """Value of every row of x from the joint Cholesky of [rows; x_i] and the same base samples z (S, |rows| + 1):
    the first `n_incumbent` rows set the incumbent, the remaining rows of `rows` are the other batch points."""
    nc = len(rows)
    z = torch.as_tensor(z, dtype=F64)
    out = torch.empty(len(x), dtype=F64)
    for i in range(len(x)):
        m, cov = oracle.posterior_joint(om, np.concatenate([rows, x[i:i + 1]]))
        L = torch.linalg.cholesky(cov)
        o = a * (m[None, :] + z @ L.T) + b
        g = o[:, :n_incumbent].amax(1)
        u = o - g[:, None]
        t = _terms(u[:, nc:], log_nei, tau_relu).T  # (1, S)
        terms = _terms(u[:, n_incumbent:nc], log_nei, tau_relu) if nc > n_incumbent else None
        out[i] = _reduce(t, terms, log_nei, tau_max)[0]
    return out


def joint_posterior_f64(gp, rows, with_beta=False):
    """Stand-in of ``baybe_b200.noisy._joint_posterior``: the oracle's joint posterior of the rows, float64, and the
    rows themselves as what ``StandInGP.cross_covariance`` takes."""
    rows = np.asarray(rows, dtype=np.float64)
    mu, cov = oracle.posterior_joint(gp.om, rows)
    return mu.numpy(), cov.numpy(), ((rows, None) if with_beta else None)


class StandInGP(OracleBackedGP):
    """OracleBackedGP plus the pending-point calls the noisy-EI scorer makes (as in tests/test_mo.py)."""

    handle = 0

    def pending_stats(self, pending):
        p = np.asarray(pending, dtype=np.float64).reshape(-1, self.d)
        mu, cov = oracle.posterior_joint(self.om, p)
        return p, None, mu.float(), cov.float()

    def cross_covariance(self, x, pend_x, beta):
        x = np.asarray(x, dtype=np.float64)
        mu, var = oracle.posterior(self.om, x)
        P = len(pend_x)
        _, cov = oracle.posterior_joint(self.om, np.concatenate([pend_x, x]))
        return mu.float(), var.float(), cov[P:, :P].float().contiguous()
