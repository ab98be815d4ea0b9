"""Float64 definitions of qLogNParEGO (test infrastructure): the arithmetic of csrc/parego.cu (``parego_values_f64`` /
``parego_score_f64``, a stand-in for ``baybe_b200::parego_score``), the value from the full joint Cholesky of [C; x]
per target (``parego_full_joint``), and stand-in models whose joint posterior is the oracle's."""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import torch

import oracle
from tests.nei_oracle import StandInGP, _reduce, _terms, joint_posterior_f64  # noqa: F401 (re-exported)

F64 = torch.float64


def _t64(v, dev=None):
    return v.detach().to(dev or v.device, F64) if torch.is_tensor(v) else torch.as_tensor(np.asarray(v), dtype=F64)


def chebyshev_t(p: torch.Tensor, alpha: float) -> torch.Tensor:
    """min_m p_m + alpha sum_m p_m over the last axis."""
    return p.amin(-1) + alpha * p.sum(-1)


def parego_values_f64(mu, var, cross, linv, w, zx, g, terms, W, V, alpha: float, tau_relu: float,
                      tau_max: float, log: bool = True, du=None) -> torch.Tensor:
    """The definition of bb_parego_score in float64: mu/var [M, N], cross [M, N, C] or None, linv [M, C, C],
    w [M, C, S] (sample-minor), zx [S, M] (the candidate's base samples per target), g [S], terms [S, Q] or None,
    p_m = W_m y_m + V_m.  With log=False the hard value mean_s max(relu(cheb_s - g_s), terms_s) instead; `du` [N]
    (error bounds only) shifts the improvement cheb_s - g_s of row i by du_i."""
    dev = mu.device if torch.is_tensor(mu) else torch.device("cpu")
    mu, var, zx, g = (_t64(v, dev).to(dev) for v in (mu, var, zx, g))
    M, N = mu.shape
    P = torch.empty(N, zx.shape[0], M, dtype=F64, device=dev)
    for m in range(M):
        if cross is not None and cross.shape[2] > 0:
            c = _t64(cross[m], dev).to(dev)
            r = c @ _t64(linv[m], dev).to(dev).T
            r2, dm = (r * r).sum(1), c @ _t64(w[m], dev).to(dev)
        else:
            r2, dm = torch.zeros_like(mu[m]), torch.zeros(N, zx.shape[0], dtype=F64, device=dev)
        sd = (var[m] - r2).clamp_min(0.0).sqrt()
        P[:, :, m] = float(W[m]) * (mu[m][:, None] + dm + sd[:, None] * zx[None, :, m]) + float(V[m])
    u = chebyshev_t(P, alpha) - g[None, :]
    if du is not None:
        u = u + du[:, None]
    return _reduce(_terms(u, log, tau_relu), terms, log, tau_max)


def parego_score_f64(mu, var, cross, linv, w, z, g, batch_terms, keep, weight, offset, params, index_offset,
                     want_scores):
    """Float64 stand-in of ``baybe_b200::parego_score`` (same arguments)."""
    from baybe_b200.engine import pack_best

    cpu = lambda v: None if v is None else v.detach().double().cpu()  # noqa: E731
    alpha, tau_relu, tau_max = params
    M = mu.shape[0]
    nc = 0 if cross is None else cross.shape[2]
    zc = cpu(z)
    zx = torch.stack([zc[:, m * (nc + 1) + nc] for m in range(M)], dim=1)
    val = parego_values_f64(cpu(mu), cpu(var), cpu(cross), cpu(linv), cpu(w), zx, cpu(g), cpu(batch_terms), weight,
                            offset, alpha, tau_relu, tau_max)
    s32 = val.float()
    best = -(1 << 63)
    for i in range(len(s32)):
        if (keep is None or int(keep[i]) != 0) and not math.isnan(float(s32[i])):
            best = max(best, pack_best(float(s32[i]), i + int(index_offset)))
    return (s32 if want_scores else None), torch.tensor([best], dtype=torch.int64)


def parego_full_joint(oms, rows: np.ndarray, n_incumbent: int, x: np.ndarray, z: np.ndarray, W, V, alpha: float,
                      tau_relu: float, tau_max: float) -> torch.Tensor:
    """Value of every row of x from the joint Cholesky of [rows; x_i] per target model and the same base samples z
    (S, M(|rows| + 1)): the first `n_incumbent` rows set the incumbent, the remaining rows of `rows` are the other
    batch points."""
    nc, M = len(rows), len(oms)
    z = torch.as_tensor(z, dtype=F64)
    out = torch.empty(len(x), dtype=F64)
    for i in range(len(x)):
        P = torch.empty(z.shape[0], nc + 1, M, dtype=F64)
        for m, om in enumerate(oms):
            mean, cov = oracle.posterior_joint(om, np.concatenate([rows, x[i:i + 1]]))
            L = torch.linalg.cholesky(cov)
            P[:, :, m] = float(W[m]) * (mean[None, :] + z[:, m * (nc + 1):(m + 1) * (nc + 1)] @ L.T) + float(V[m])
        cheb = chebyshev_t(P, alpha)
        u = cheb - cheb[:, :n_incumbent].amax(1, keepdim=True)
        t = _terms(u[:, nc:], True, tau_relu).T  # (1, S)
        terms = _terms(u[:, n_incumbent:nc], True, tau_relu) if nc > n_incumbent else None
        out[i] = _reduce(t, terms, True, tau_max)[0]
    return out


def stand_in_models(w, n_targets: int, noise: float = 1e-2, seed: int = 0):
    """One oracle-backed model per target on the rows of workload `w`: target m measures a different smooth
    function of the same rows (``StandInGP``, its measurements kept as ``train_y``)."""
    from baybe_b200.synthetic import smooth_target

    gps = []
    for m in range(n_targets):
        y = smooth_target(w.train_x, seed=seed + 7 * m + 1)
        gps.append(StandInGP(**dataclasses.replace(w, train_y=y, noise=np.array([noise])).gp_kwargs()))
        gps[-1].train_y = y
    return gps
