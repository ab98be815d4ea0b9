"""Float64 value and gradient of the single-target acquisition functions by torch autograd of the oracle's torch
pieces (test infrastructure only): the reference for ``bb_acq_grad`` and, behind the ``value_and_grad`` seam, the
stand-in engine of the CPU tests of ``baybe_b200.continuous``.

``oracle.posterior`` converts its input with ``np.asarray``, which cuts the autograd graph, so the value is built here
from ``_normalise``, ``kernel_matrix``, ``_standardised_posterior``, ``acq_from_moments`` and the candidate-first
Cholesky form of ``acq_values_joint``, with a leaf tensor for X."""
from __future__ import annotations

import math

import numpy as np
import torch

import oracle
from oracle import reference_path as rp
from tests.helpers import OracleBackedGP


def oracle_moments(om, X: torch.Tensor, pending=None):
    """Differentiable float64 mean [B], variance [B] and, with pending points, the pending means [p], covariance
    [p, p] and cross covariance [B, p] (original units)."""
    Xn = rp._normalise(X, om.lo, om.rng)
    _, m, V = rp._standardised_posterior(om, Xn)
    var_s = (rp._kernel_diag(om.spec, Xn) - (V * V).sum(-1)).clamp_min(rp.MIN_VARIANCE)
    mu = om.y_mean + om.y_std * m
    var = om.y_std**2 * var_s
    P = None if pending is None else torch.as_tensor(np.asarray(pending), dtype=torch.float64).reshape(-1, X.shape[1])
    if P is None or len(P) == 0:
        return mu, var, None
    s2 = om.y_std**2
    Pn = rp._normalise(P, om.lo, om.rng)
    _, mP, VP = rp._standardised_posterior(om, Pn)
    covPP = rp.kernel_matrix(om.spec, Pn, Pn) - VP @ VP.T
    covPP.diagonal().copy_(rp._kernel_diag(om.spec, Pn) - (VP * VP).sum(-1))
    cross = s2 * (rp.kernel_matrix(om.spec, Xn, Pn) - V @ VP.T)
    return mu, var, (om.y_mean + om.y_std * mP, s2 * covPP, cross)


def _log_fatplus(x: torch.Tensor, tau: float) -> torch.Tensor:
    """``reference_path._log_fatplus`` with the same values and a finite gradient everywhere: its unselected branch
    takes log(0) for very negative t, whose gradient turns the selected one's into NaN (inf * 0)."""
    t = x / tau
    t_safe = torch.where(t < -30.0, torch.zeros_like(t), t)
    log_sp = torch.where(t < -30.0, t, torch.log(torch.nn.functional.softplus(t_safe)))
    log_cauchy = math.log(rp.FATPLUS_ALPHA) - torch.log1p(t * t)
    return math.log(tau) + torch.logaddexp(log_sp, log_cauchy)


def _mc_reduce(acq, obj: torch.Tensor) -> torch.Tensor:
    if acq.kind != "qLogEI":
        return rp._mc_reduce(acq, obj, None)
    li = _log_fatplus(obj - acq.best_f, acq.tau_relu)
    li = rp._fatmax(li, acq.tau_max, dim=-1) if obj.shape[-1] > 1 else li.squeeze(-1)
    return torch.logsumexp(li, dim=0) - math.log(obj.shape[0])


def acq_of_moments(acq: "oracle.AcqSpec", mu, var, pend=None, z=None) -> torch.Tensor:
    """Acquisition values from the moments of ``oracle_moments`` (with pending points: candidate-first Cholesky)."""
    if pend is None:
        if not acq.is_mc:
            return rp._analytic(acq, mu, var)
        zz = torch.as_tensor(z, dtype=torch.float64).reshape(-1, 1)
        return _mc_reduce(acq, (acq.obj_scale * (mu.unsqueeze(0) + var.sqrt().unsqueeze(0) * zz)
                                + acq.obj_shift).unsqueeze(-1))
    mP, covPP, cross = pend
    z = torch.as_tensor(z, dtype=torch.float64)
    B, p = cross.shape
    top = torch.cat([var.unsqueeze(-1), cross], dim=-1).unsqueeze(1)                    # (B,1,1+p)
    bot = torch.cat([cross.unsqueeze(-1), covPP.expand(B, p, p)], dim=-1)              # (B,p,1+p)
    cov = torch.cat([top, bot], dim=1)
    mean = torch.cat([mu.unsqueeze(-1), mP.unsqueeze(0).expand(B, p)], dim=-1)
    L = rp._chol_with_jitter(cov)
    y = mean.unsqueeze(0) + torch.einsum("bij,sj->sbi", L, z)
    return _mc_reduce(acq, acq.obj_scale * y + acq.obj_shift)


def oracle_value(om, acq: "oracle.AcqSpec", X: torch.Tensor, z=None, pending=None) -> torch.Tensor:
    """Differentiable float64 acquisition values of the rows of X (with pending points: of [x; pending])."""
    mu, var, pend = oracle_moments(om, X, pending)
    return acq_of_moments(acq, mu, var, pend, z)


def oracle_value_and_grad(om, acq, X, z=None, pending=None) -> tuple[torch.Tensor, torch.Tensor]:
    Xl = torch.as_tensor(np.asarray(X), dtype=torch.float64).clone().requires_grad_(True)
    val = oracle_value(om, acq, Xl, z, pending)
    (g,) = torch.autograd.grad(val.sum(), Xl)
    return val.detach(), g


class OracleGradGP(OracleBackedGP):
    """``OracleBackedGP`` with ``value_and_grad`` (``DeviceGP``'s signature) from float64 autograd of the oracle."""

    def value_and_grad(self, acq, x, z, pending=None):
        v, g = oracle_value_and_grad(self.om, self._spec(acq), torch.as_tensor(np.asarray(x), dtype=torch.float64),
                                     z, pending)
        return v.float(), g.float()
