"""Float64 value and gradient of ``bb_hvi_grad`` by torch autograd of a literal restatement of its definition (test
infrastructure only): the reference of the GPU tests and, behind the ``multiobjective._hvi_grad`` seam, the stand-in
engine of the CPU tests of qEHVI / qLogEHVI on continuous and hybrid search spaces.

Per point x, target m and base sample s (csrc/mo.cu, csrc/hvigrad.cu):
    y_ms = a_m (mu_m + c_m . w_ms + sd_m z_ms) + b_m,   sd_m = sqrt(max(var_m - |L_m^-1 c_m|^2, 0))
    h_s  = ``mo_oracle.cell_values`` of y_s over the cells of the one decomposition (no pending points) or of sample
           s's decomposition,   A = mean_s h_s (qEHVI) or logmeanexp_s h_s (qLogEHVI).
mu_m, var_m and c_m come from the oracle's posterior of x (``continuous_oracle.oracle_moments``); L_m^-1, w and the
cells are the given constants of the step's conditioning.  ``cell_values`` runs with continuous_oracle's log fatplus,
which has the same values and a finite gradient where the reference's takes log(0) in its unselected branch."""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import mo_oracle
from tests.continuous_oracle import _log_fatplus, oracle_moments
from tests.objective_grad_oracle import StandInObjectiveGP


def cell_values(Y: torch.Tensor, lower, upper, log: bool, tau_relu: float, tau_max: float) -> torch.Tensor:
    """``mo_oracle.cell_values`` with a log fatplus whose gradient is finite everywhere."""
    saved = mo_oracle._log_fatplus
    mo_oracle._log_fatplus = _log_fatplus
    try:
        return mo_oracle.cell_values(Y, lower, upper, log, tau_relu, tau_max)
    finally:
        mo_oracle._log_fatplus = saved


def samples(moments, linv, w, z, a, b) -> torch.Tensor:
    """The oriented conditional samples y [S, B, M] from every target's (mu, var, pending) moments."""
    z = torch.as_tensor(z).double()
    M = len(moments)
    Q = z.shape[1] // M
    P = Q - 1
    ys = []
    for m, (mu, var, pend) in enumerate(moments):
        zx = z[:, m * Q + P]
        if P == 0:
            y = mu[None] + var.clamp_min(0).sqrt()[None] * zx[:, None]
        else:
            c = pend[2]                                                    # (B, P)
            r = c @ torch.as_tensor(linv[m]).double().T
            sd = (var - (r * r).sum(-1)).clamp_min(0).sqrt()
            y = mu[None] + torch.as_tensor(w[m]).double() @ c.T + sd[None] * zx[:, None]
        ys.append(float(a[m]) * y + float(b[m]))
    return torch.stack(ys, -1)


def hvi_value(moments, linv, w, z, lower, upper, n_cells, log: bool, a, b, tau_relu: float, tau_max: float):
    """Differentiable float64 value [B] (what ``bb_hvi_grad`` writes) from the targets' moments."""
    Y = samples(moments, linv, w, z, a, b)
    S = Y.shape[0]
    lower = torch.as_tensor(lower).double()
    upper = torch.as_tensor(upper).double()
    n_cells = [int(v) for v in torch.as_tensor(n_cells).reshape(-1)]
    if lower.shape[0] == 1:
        v = cell_values(Y, lower[0, :n_cells[0]], upper[0, :n_cells[0]], log, tau_relu, tau_max)
    else:
        v = torch.stack([cell_values(Y[s], lower[s, :n_cells[s]], upper[s, :n_cells[s]], log, tau_relu, tau_max)
                         for s in range(S)])
    return (torch.logsumexp(v, 0) - math.log(S)) if log else v.mean(0)


def hvi_grad_f64(gps, x, pend_x, betas, linv, w, z, lower, upper, n_cells, kind, params, a, b):
    """Float64 stand-in of ``baybe_b200::hvi_grad`` (the arguments of the ``multiobjective._hvi_grad`` seam: the
    models, then those of the op) -> (value [N], gradient [N, d]) as float32."""
    from baybe_b200.engine import AcqConfig

    cfg = AcqConfig.from_params(kind, params)
    cpu = (lambda t: None if t is None else (t.detach().double().cpu() if torch.is_tensor(t) else
                                             torch.as_tensor(np.asarray(t), dtype=torch.float64)))
    X = cpu(x).clone().requires_grad_(True)
    px = cpu(pend_x)
    moments = [oracle_moments(gp.om, X, px) for gp in gps]
    val = hvi_value(moments, cpu(linv), cpu(w), cpu(z), cpu(lower), cpu(upper), n_cells.cpu(),
                    cfg.kind == "qLogEHVI", a, b, cfg.tau_relu, cfg.tau_max)
    (g,) = torch.autograd.grad(val.sum(), X)
    return val.detach().float(), g.float()


StandInHviGP = StandInObjectiveGP  # pending statistics and cross covariances from the oracle
