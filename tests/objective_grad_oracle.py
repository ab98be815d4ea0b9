"""Float64 value and gradient of ``bb_objective_grad`` by torch autograd of a literal restatement of its definition
(test infrastructure only): the reference of the GPU tests and, behind the ``objectives._objective_grad`` seam, the
stand-in engine of the CPU tests of the continuous and hybrid paths for desirability and transformed targets.

Per point x, target m and base sample s (csrc/objective.cu, csrc/objgrad.cu):
    y_ms = mu_m + c_m . w_ms + sd_m z_ms,   sd_m = sqrt(max(var_m - |L_m^-1 c_m|^2, 0))
    t_ms = program_m(y_ms),   o_s = scalarise(t_s),   A = acquisition over o_s joined with the pending terms
mu_m, var_m and c_m come from the oracle's posterior of x (``continuous_oracle.oracle_moments``); L_m^-1, w and the
pending terms are the given constants of the step's conditioning.  A max passes its gradient to its first maximal
entry, the candidate first (torch.argmax + gather)."""
from __future__ import annotations

import math

import numpy as np
import torch

import oracle
from oracle import reference_path as rp
from tests.continuous_oracle import _log_fatplus, oracle_moments
from tests.helpers import OracleBackedGP
from tests.objective_oracle import _programs, objective


def _first_max(x: torch.Tensor) -> torch.Tensor:
    return x.gather(-1, x.argmax(-1, keepdim=True))


def _fatmax_first(x: torch.Tensor, tau: float) -> torch.Tensor:
    """botorch fatmax with its hard maximum taken as the first maximal entry."""
    M = _first_max(x)
    par = (1.0 + (M - x) / (tau * rp.FATMAX_ALPHA)).pow(-rp.FATMAX_ALPHA)
    return (M + tau * par.sum(-1, keepdim=True).log()).squeeze(-1)


def _terms(cfg, o: torch.Tensor) -> torch.Tensor:
    if cfg.kind == "qLogEI":
        return _log_fatplus(o - cfg.best_f, cfg.tau_relu)
    if cfg.kind == "qEI":
        return (o - cfg.best_f).clamp_min(0.0)
    if cfg.kind == "qPI":
        return torch.sigmoid((o - cfg.best_f) / cfg.tau_pi)
    if cfg.kind == "qSR":
        return o
    m = o.mean(0, keepdim=True)
    return m + math.sqrt(cfg.beta * math.pi / 2) * (o - m).abs()


def objective_value(oms, X: torch.Tensor, pend_x, linv, w, pend_terms, z, cfg, progs, scal: str, weights):
    """Differentiable float64 acquisition values [B] of the rows of X (one oracle model per target)."""
    M = len(oms)
    P = 0 if pend_x is None else len(pend_x)
    px = None if P == 0 else torch.as_tensor(np.asarray(pend_x), dtype=torch.float64)
    moments = [oracle_moments(om, X, px) for om in oms]
    if not cfg.is_mc:  # MEAN over affine targets: Gaussian moments
        a = [p[0][1][0] if p else 1.0 for p in progs]
        b = [p[0][1][1] if p else 0.0 for p in progs]
        mean = sum(weights[m] * (a[m] * moments[m][0] + b[m]) for m in range(M))
        var = sum((weights[m] * a[m]) ** 2 * moments[m][1] for m in range(M))
        acq = oracle.AcqSpec(kind=cfg.kind, best_f=cfg.best_f, beta=cfg.beta, maximize=cfg.maximize)
        return rp._analytic(acq, mean, var)
    z = torch.as_tensor(z).double()
    Q = P + 1
    ys = []
    for m, (mu, var, pend) in enumerate(moments):
        zx = z[:, m * Q + P]
        if P == 0:
            ys.append(mu[None] + var.clamp_min(0).sqrt()[None] * zx[:, None])
            continue
        c = pend[2]                                                        # (B, P)
        r = c @ torch.as_tensor(linv[m]).double().T
        sd = (var - (r * r).sum(-1)).clamp_min(0).sqrt()
        ys.append(mu[None] + torch.as_tensor(w[m]).double() @ c.T + sd[None] * zx[:, None])
    o = objective(progs, scal, weights, torch.stack(ys, -1))                # (S, B)
    tx = _terms(cfg, o)
    S = o.shape[0]
    if P:
        pt = torch.as_tensor(pend_terms).double()
        allt = torch.cat([tx[:, :, None], pt[:, None, :].expand(-1, tx.shape[1], -1)], -1)
        tx = _fatmax_first(allt, cfg.tau_max) if cfg.kind == "qLogEI" else _first_max(allt).squeeze(-1)
    if cfg.kind == "qLogEI":
        return torch.logsumexp(tx, 0) - math.log(S)
    return tx.mean(0)


def objective_grad_f64(gps, x, pend_x, betas, linv, w, pend_terms, z, kind, params, scalarizer, ops, args, n_ops,
                       weights):
    """Float64 stand-in of ``baybe_b200::objective_grad`` (the arguments of the ``objectives._objective_grad`` seam:
    the models, then those of the op) -> (value [N], gradient [N, d]) as float32."""
    from baybe_b200 import _lib
    from baybe_b200.engine import AcqConfig

    cfg = AcqConfig.from_params(kind, params)
    scal = {v: k for k, v in _lib.OBJ_SCALARIZER.items()}[scalarizer]
    progs = _programs(ops, args, n_ops)
    cpu = (lambda t: None if t is None else (t.detach().double().cpu() if torch.is_tensor(t) else
                                             torch.as_tensor(np.asarray(t), dtype=torch.float64)))
    X = cpu(x).clone().requires_grad_(True)
    val = objective_value([gp.om for gp in gps], X, cpu(pend_x), cpu(linv), cpu(w), cpu(pend_terms), cpu(z), cfg,
                          progs, scal, [float(v) for v in weights])
    if val.requires_grad:
        (g,) = torch.autograd.grad(val.sum(), X)
    else:  # the objective does not depend on x (a CONST program)
        g = torch.zeros_like(X)
    return val.detach().float(), g.float()


class StandInObjectiveGP(OracleBackedGP):
    """``OracleBackedGP`` with the pending-point statistics ``ObjectiveScorer`` needs (tests/test_objectives.py's
    stand-in)."""

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
