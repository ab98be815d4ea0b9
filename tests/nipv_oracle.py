"""Float64 definitions of qNIPV (test infrastructure): the arithmetic of csrc/nipv.cu from the op's own inputs
(``nipv_score_f64``, a stand-in for ``baybe_b200::nipv_score``), the value straight from the joint posterior with
explicit noisy conditioning (``nipv_definition``), and an engine stand-in whose posterior is the oracle's."""
from __future__ import annotations

import itertools
import math
from types import SimpleNamespace

import numpy as np
import torch

import oracle
from tests.helpers import OracleBackedGP

_REGISTRY: dict[int, "NipvStandInGP"] = {}
_HANDLES = itertools.count(1)


class NipvStandInGP(OracleBackedGP):
    """OracleBackedGP with what ``NipvScorer`` reads of a ``DeviceGP``: float64 posteriors, the hyper-parameters by
    name and a handle under which ``nipv_score_f64`` finds the model."""

    def __init__(self, train_x, train_y, bounds, family, lengthscale, noise, mean_const=0.0, outputscale=None,
                 task_col=None, task_covar=None, device=None):
        super().__init__(train_x, train_y, bounds, family, lengthscale, noise, mean_const, outputscale, task_col,
                         task_covar, device)
        T = 1 if task_covar is None else int(np.asarray(task_covar).shape[0])
        self.task_col, self.n_tasks, self.outputscale = task_col, T, outputscale
        self.task_covar = None if task_covar is None else np.asarray(task_covar, dtype=np.float64)
        self.noise = np.broadcast_to(np.asarray(noise, dtype=np.float64), (T,)).copy()
        self.model = SimpleNamespace(y_std=float(self.om.y_std), wide=0)
        self.handle = next(_HANDLES)
        _REGISTRY[self.handle] = self

    def posterior(self, x):
        return oracle.posterior(self.om, np.asarray(x, dtype=np.float64))

    def cross_covariance(self, x, pend_x, beta):
        x = np.asarray(x, dtype=np.float64)
        mu, var = oracle.posterior(self.om, x)
        P = len(pend_x)
        _, cov = oracle.posterior_joint(self.om, np.concatenate([np.asarray(pend_x, dtype=np.float64), x]))
        return mu, var, cov[P:, :P].contiguous()

    def noise_orig(self, rows: np.ndarray) -> np.ndarray:
        """Likelihood noise of each row (its task's, floored at 1e-4) in original units."""
        t = np.zeros(len(rows), dtype=np.int64) if self.task_col is None else np.clip(
            np.rint(rows[:, self.task_col]).astype(np.int64), 0, self.n_tasks - 1)
        return np.maximum(self.noise[t], 1e-4) * float(self.om.y_std) ** 2


def joint_posterior_f64(gp, rows, with_beta=False):
    """Stand-in of ``baybe_b200.noisy._joint_posterior``: the oracle's joint posterior of the rows, float64, and the
    rows themselves as what ``NipvStandInGP.cross_covariance`` takes."""
    rows = np.asarray(rows, dtype=np.float64)
    mu, cov = oracle.posterior_joint(gp.om, rows)
    return mu.numpy(), cov.numpy(), ((rows, None) if with_beta else None)


def nipv_score_f64(x, xm, var, cross_x, cross_m, linv, keep, handle, index_offset, want_scores):
    """Float64 stand-in of ``baybe_b200::nipv_score`` (same arguments): IVR(x) = sum_m k_C(m,x)^2 / (k_C(x,x) +
    noise(x)) with k_C(m,x) = k_D(m,x) - (L_C^-1 c_m) . (L_C^-1 c_x), k_C(x,x) = var - |L_C^-1 c_x|^2."""
    from baybe_b200.engine import pack_best

    gp = _REGISTRY[handle]
    X, XM = x.detach().double().cpu().numpy(), xm.detach().double().cpu().numpy()
    M = len(XM)
    _, cov = oracle.posterior_joint(gp.om, np.concatenate([XM, X]))
    kmx = cov.numpy()[:M, M:]
    kxx = var.detach().double().cpu().numpy()
    if cross_x is not None:
        L = linv.detach().double().cpu().numpy()
        ax = cross_x.detach().double().cpu().numpy() @ L.T
        am = cross_m.detach().double().cpu().numpy() @ L.T
        kmx = kmx - am @ ax.T
        kxx = kxx - (ax * ax).sum(1)
    ivr = torch.from_numpy((kmx * kmx).sum(0) / (kxx + gp.noise_orig(X)))
    best = -(1 << 63)
    for i, v in enumerate(ivr.float().tolist()):
        if (keep is None or int(keep[i]) != 0) and not math.isnan(v):
            best = max(best, pack_best(v, i + int(index_offset)))
    return (ivr if want_scores else None), torch.tensor([best], dtype=torch.int64)


def nipv_definition(gp, X: np.ndarray, XM: np.ndarray, C: np.ndarray) -> np.ndarray:
    """-(1/M) sum_m Var[f(m) | D, y(x), y(C)] for every row x of X, original units, float64: the joint posterior of
    [XM; x; C] from the oracle, conditioned on noisy observations of [x; C]."""
    out = np.empty(len(X))
    M = len(XM)
    for i, x in enumerate(X):
        rows = np.concatenate([XM, x[None, :], C])
        cov = oracle.posterior_joint(gp.om, rows)[1].numpy()
        S = slice(M, len(rows))
        K = cov[S, S] + np.diag(gp.noise_orig(rows[S]))
        red = (cov[:M, S] @ np.linalg.solve(K, cov[S, :M])).diagonal()
        out[i] = -float((np.diag(cov)[:M] - red).sum()) / M
    return out


def batch_definition(gp, rows: np.ndarray, XM: np.ndarray) -> float:
    """-(1/M) sum_m Var[f(m) | D, y(rows)]: the joint value of a q-batch (pending points included in `rows`)."""
    return float(nipv_definition(gp, rows[:1], XM, rows[1:])[0])
