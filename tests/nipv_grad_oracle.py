"""Float64 value and gradient of ``bb_nipv_grad`` by torch autograd of a literal restatement of qNIPV's definition (test
infrastructure only): the reference of the GPU tests and, behind the ``nipv._nipv_phi`` / ``nipv._nipv_grad`` seams,
the stand-in engine of the CPU tests of qNIPV on continuous and hybrid spaces.

For a point x, integration points XM and conditioning rows C, with Var[. | D, y(S)] the posterior variance given the
training data and noisy observations of the rows S (``oracle.posterior_joint``'s covariance of [XM; C; x], then the
Gaussian conditioning on y(S)):
    IVR(x) = sum_m ( Var[f(m) | D, y(C)] - Var[f(m) | D, y(C), y(x)] )          (original units)
and qNIPV(x | C) = -(1/M) sum_m Var[f(m) | D, y(C), y(x)] (``nipv_oracle.nipv_definition``)."""
from __future__ import annotations

import numpy as np
import torch

from oracle import reference_path as rp
from tests.nipv_oracle import _REGISTRY


def joint_cov(om, rows: torch.Tensor) -> torch.Tensor:
    """``oracle.posterior_joint``'s covariance (original units), differentiable in the rows."""
    Xn = rp._normalise(rows, om.lo, om.rng)
    _, _, V = rp._standardised_posterior(om, Xn)
    cov = rp.kernel_matrix(om.spec, Xn, Xn) - V @ V.T
    cov = cov - torch.diag(cov.diagonal()) + torch.diag(rp._kernel_diag(om.spec, Xn) - (V * V).sum(-1))
    return om.y_std**2 * cov


def ivr_definition(om, noise_orig, X: torch.Tensor, XM: np.ndarray, C: np.ndarray | None,
                   chunk: int = 4096) -> torch.Tensor:
    """IVR(x) [P] of the rows of X (float64, differentiable in X) under the oracle model `om`, given the integration
    rows XM (taken `chunk` at a time: the sum over m splits) and the conditioning rows C (None: empty);
    `noise_orig(rows)`: the likelihood noise of each row in original units."""
    Cn = 0 if C is None else len(C)
    P = len(X)
    Crows = np.asarray(C, dtype=np.float64).reshape(Cn, -1) if Cn else np.zeros((0, X.shape[1]))
    noise = torch.as_tensor(noise_orig(np.concatenate([Crows, X.detach().numpy()])), dtype=torch.float64)
    total = torch.zeros(P, dtype=torch.float64)
    for m0 in range(0, len(XM), chunk):
        xm = np.asarray(XM[m0:m0 + chunk], dtype=np.float64)
        M = len(xm)
        cov = joint_cov(om, torch.cat([torch.as_tensor(np.concatenate([xm, Crows])), X]))

        def reduction(S: list[int]) -> torch.Tensor:  # sum_m of the variance that y(S) takes away at m
            if not S:
                return torch.zeros((), dtype=torch.float64)
            K = cov[S][:, S] + torch.diag(noise[[s - M for s in S]])
            B = cov[:M][:, S]
            return (B * torch.linalg.solve(K, B.T).T).sum()

        cs = list(range(M, M + Cn))
        base = reduction(cs)
        total = total + torch.stack([reduction(cs + [M + Cn + i]) - base for i in range(P)])
    return total


def nipv_phi_f64(xm, cross_m, linv, handle):
    """Stand-in of ``baybe_b200::nipv_phi``: its "image" is the integration rows themselves, float64, from which
    ``nipv_grad_f64`` recomputes everything."""
    return xm.detach().double().cpu().reshape(-1).clone()


def nipv_grad_f64(x, img, M, cond_x, cond_beta, linv, handle):
    """Stand-in of ``baybe_b200::nipv_grad`` (same arguments): IVR [P] (original units) and its gradient [P, d] by
    autograd of ``ivr_definition``; the conditioning rows come as ``nipv_oracle.joint_posterior_f64`` gives them."""
    gp = _REGISTRY[handle]
    X = torch.as_tensor(x.detach().cpu().numpy(), dtype=torch.float64).requires_grad_(True)
    C = None if cond_x is None else np.asarray(cond_x, dtype=np.float64)
    ivr = ivr_definition(gp.om, gp.noise_orig, X, img.reshape(M, -1).numpy(), C)
    g = torch.autograd.grad(ivr.sum(), X)[0] if X.shape[0] else torch.zeros_like(X)
    return ivr.detach(), g
