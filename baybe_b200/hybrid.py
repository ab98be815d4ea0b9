"""Hybrid (discrete x continuous) recommendation on the device -- SURVEY.md 8f-2, BASELINE config 3.

Replaces ``recommend_hybrid_without_subsets`` (``/root/reference/baybe/recommenders/pure/bayesian/botorch/hybrid.py:30-161``):
the reference fixes every discrete configuration in turn and runs ``optimize_acqf_mixed`` -- sequential greedy over
the batch, and for each discrete configuration a multi-start L-BFGS over the continuous parameters
(``hybrid.py:110``) on an acquisition function built by ``acquisition/_builder.py:195-334`` (``X_baseline`` = the
training inputs for the noisy-EI family, ``:319-324``).

Design: no gradient ascent.  The scoring path runs at 10^8-10^9 candidates per second, so a greedy step
is a *search by scoring*: every discrete configuration x a shared scrambled-Sobol set of continuous points is scored
in one sweep, the best seeds are refined by sweeps over shrinking boxes, and the winner joins the pending set.  The
result is deterministic for a seed and is judged the way a stochastic multi-start optimiser has to be: by the
acquisition value of the recommended batch (tests compare it with an exhaustive oracle search).

qNEI (``acquisition/acqfs.py:227-232``) is evaluated in its conditional form.  With C = [baseline; pending] and the
joint Cholesky taken in the order [C; x],
    f_x,s = mu_x + r_x . Z_C[s] + sqrt(var_x - |r_x|^2) z_x,s,   r_x = Sigma_xC L_C^-T,
    value(x) = mean_s relu(o(f_x,s) - g_s),   g_s = max_C o(f_C,s)
so one sweep over N candidates is: K(X, X_train) (``bb_kernel_matrix``, hand-written), the posterior
moments and the covariance with the pending points (``bb_posterior``), ONE dense GEMM Sigma_XC @ [W | L_C^-T]
(cuBLAS through ``torch.matmul``: a plain library GEMM) and ``bb_nei_reduce`` (hand-written).  The m x m setup
(posterior covariance of C, its Cholesky, W = L_C^-T Z_C^T) is float64 torch on the device, once per greedy step.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.acquisition import AcqConfig
from baybe_b200.engine import DeviceGP, sobol_normal_samples

__all__ = ["NeiScorer", "HybridSearch", "recommend_hybrid"]

_SQRT5, _SQRT3 = math.sqrt(5.0), math.sqrt(3.0)


def _kernel64(family: str, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """float64 stationary kernel of pre-scaled rows (x / lengthscale), as gpytorch evaluates it."""
    d2 = (a * a).sum(-1, keepdim=True) + (b * b).sum(-1).unsqueeze(0) - 2.0 * a @ b.T
    d2 = d2.clamp_min(0.0)
    if family == "rbf":
        return torch.exp(-0.5 * d2)
    r = d2.sqrt()
    if family == "matern12":
        return torch.exp(-r)
    if family == "matern32":
        return (1.0 + _SQRT3 * r) * torch.exp(-_SQRT3 * r)
    return (1.0 + _SQRT5 * r + (5.0 / 3.0) * d2) * torch.exp(-_SQRT5 * r)


def _psd_cholesky(cov: torch.Tensor) -> torch.Tensor:
    """linear_operator ``psd_safe_cholesky``: plain attempt, then jitter 1e-8 * 10^i (float64)."""
    L, info = torch.linalg.cholesky_ex(cov)
    if int(info) == 0:
        return L
    for i in range(3):
        L, info = torch.linalg.cholesky_ex(cov + (1e-8 * 10**i) * torch.eye(cov.shape[0], dtype=cov.dtype, device=cov.device))
        if int(info) == 0:
            return L
    raise FloatingPointError("joint covariance of the conditioning set is not positive definite")


class NeiScorer:
    """qNEI marginal gains of single new points given a pending set, for a fitted single-task ``DeviceGP``."""

    BLOCK = 65536  # candidate rows per GEMM block: 65536 x (S + m) floats of workspace

    def __init__(self, gp: DeviceGP, acq: AcqConfig, n_samples: int = 512, seed: int = 0):
        if gp.task_col is not None:
            raise NotImplementedError("qNEI on the device supports single-task models")
        self.gp, self.acq, self.S, self.seed = gp, acq, int(n_samples), int(seed)
        dev = gp.device
        tx, ty, bnd, ls, nz, mc, _ = gp._keepalive
        f64 = dict(dtype=torch.float64, device=dev)
        self.lo = torch.as_tensor(bnd[0], **f64)
        rng = torch.as_tensor(bnd[1] - bnd[0], **f64)
        self.rng = torch.where(rng.abs() < 1e-8, torch.ones_like(rng), rng)
        act = torch.as_tensor(ls > 0, device=dev)
        self.inv_ls = torch.where(act, 1.0 / torch.as_tensor(np.where(ls > 0, ls, 1.0), **f64), torch.zeros(len(ls), **f64))
        y = torch.as_tensor(ty, **f64)
        self.y_mean = float(y.mean())
        ys = float(y.std(unbiased=True)) if len(ty) > 1 else 1.0
        self.y_std = ys if ys >= 1e-8 else 1.0
        self.noise = max(float(nz[0]), 1e-4)
        self.mean_const = float(mc[0])
        self.out_scale = float(gp.outputscale) if gp.outputscale is not None else 1.0
        self.Xb = self._scaled(torch.as_tensor(tx, **f64))
        n = self.Xb.shape[0]
        K = self.out_scale * _kernel64(gp.family, self.Xb, self.Xb)
        K.diagonal().fill_(self.out_scale)
        self.Lt = _psd_cholesky(K + self.noise * torch.eye(n, **f64))
        resid = (y - self.y_mean) / self.y_std - self.mean_const
        self.alpha = torch.cholesky_solve(resid.unsqueeze(-1), self.Lt).squeeze(-1)
        KinvK = torch.cholesky_solve(K, self.Lt)  # Ktilde^-1 K
        self.Sbb = (K - K @ KinvK) * self.y_std**2  # posterior covariance of the latent at the training inputs
        self.Mb = (torch.eye(n, **f64) - KinvK) * self.y_std**2  # Sigma_Xb = K*_X @ Mb
        self.mu_b = self.y_mean + self.y_std * (self.mean_const + K @ self.alpha)
        self.n = n
        self._pending = torch.empty(0, gp.d, **f64)
        self._stale = True

    # -- small float64 helpers ---------------------------------------------------------------------------------
    def _scaled(self, x_raw: torch.Tensor) -> torch.Tensor:
        return (x_raw - self.lo) / self.rng * self.inv_ls

    def set_pending(self, pending) -> None:
        p = torch.as_tensor(np.asarray(pending, dtype=np.float64), dtype=torch.float64, device=self.gp.device)
        self._pending = p.reshape(-1, self.gp.d)
        self._stale = True

    def _setup(self) -> None:
        """Conditioning set C = [baseline; pending]: posterior moments, Cholesky, sample-dependent constants."""
        gp, dev = self.gp, self.gp.device
        P = self._pending
        p = P.shape[0]
        m = self.n + p
        z = sobol_normal_samples(self.S, m + 1, self.seed).to(dev, torch.float64)  # columns: baseline, pending, new point
        self.z = z
        cov = torch.empty(m, m, dtype=torch.float64, device=dev)
        cov[: self.n, : self.n] = self.Sbb
        mu_c = torch.empty(m, dtype=torch.float64, device=dev)
        mu_c[: self.n] = self.mu_b
        if p:
            Ps = self._scaled(P)
            kpb = self.out_scale * _kernel64(gp.family, Ps, self.Xb)  # (p, n)
            kpp = self.out_scale * _kernel64(gp.family, Ps, Ps)
            kpp.diagonal().fill_(self.out_scale)
            sol = torch.cholesky_solve(kpb.T, self.Lt)  # Ktilde^-1 k(b, P): (n, p)
            cov[self.n :, self.n :] = (kpp - kpb @ sol) * self.y_std**2
            cpb = kpb @ self.Mb  # k_pb (I - Ktilde^-1 K) y_std^2
            cov[self.n :, : self.n] = cpb
            cov[: self.n, self.n :] = cpb.T
            mu_c[self.n :] = self.y_mean + self.y_std * (self.mean_const + kpb @ self.alpha)
        Lc = _psd_cholesky(cov)
        Zc = z[:, :m]
        Fc = mu_c.unsqueeze(0) + Zc @ Lc.T  # (S, m) joint samples of C
        oc = self.acq.obj_scale * Fc + self.acq.obj_shift
        best = oc[:, : self.n].amax(-1)
        pend = oc[:, self.n :].amax(-1) if p else torch.full_like(best, -float("inf"))
        self.g = torch.maximum(best, pend).to(torch.float32).contiguous()
        self.const = float((pend - best).clamp_min(0.0).mean()) if p else 0.0
        eye = torch.eye(m, dtype=torch.float64, device=dev)
        LinvT = torch.linalg.solve_triangular(Lc, eye, upper=False).T  # L_C^-T
        W = LinvT @ Zc.T  # (m, S)
        big = torch.cat([W, LinvT], dim=1)  # (m, S + m)
        self.Gb = (self.Mb @ big[: self.n]).to(torch.float32).contiguous()  # (n, S + m): multiplies K*_X
        self.Gp = big[self.n :].to(torch.float32).contiguous()  # (p, S + m): multiplies the pending cross-covariance
        self.zx = z[:, m].to(torch.float32).contiguous()
        self.m, self.p = m, p
        if p:
            self.pend_x, self.pend_beta, _, _ = gp.pending_stats(P.to(torch.float32))
        self._stale = False

    # -- the sweep ---------------------------------------------------------------------------------------------
    def score(self, x: torch.Tensor) -> torch.Tensor:
        """Marginal qNEI gain of every row of x (fp32 row-major on the device) given the pending set; add
        ``self.const`` for the joint value of [x; pending]."""
        if self._stale:
            self._setup()
        gp, lib = self.gp, _lib.load()
        x = gp.prepare(x)
        N = x.shape[0]
        out = torch.empty(N, dtype=torch.float32, device=gp.device)
        ld = self.S + self.m
        for lo in range(0, N, self.BLOCK):
            xb = x[lo : lo + self.BLOCK]
            nb = xb.shape[0]
            ks = gp.kernel_matrix(xb)[:, : self.n]
            if self.p:
                mu, var, cross = gp.cross_covariance(xb, self.pend_x, self.pend_beta)
            else:
                mu, var = gp.posterior(xb)
                cross = None
            buf = ks @ self.Gb  # cuBLAS: (nb, n) x (n, S + m)
            if cross is not None:
                buf.addmm_(cross, self.Gp)
            with torch.cuda.device(gp.device):
                _lib.check(lib.bb_nei_reduce(
                    C.c_void_p(buf.data_ptr()), ld, self.S, self.m, C.c_void_p(mu.data_ptr()), C.c_void_p(var.data_ptr()),
                    C.c_void_p(self.zx.data_ptr()), C.c_void_p(self.g.data_ptr()), C.c_float(self.acq.obj_scale),
                    C.c_float(self.acq.obj_shift), nb, C.c_void_p(out[lo : lo + nb].data_ptr()),
                    C.c_void_p(torch.cuda.current_stream().cuda_stream)), "bb_nei_reduce")
        return out


@dataclass
class HybridSearch:
    """Search-by-scoring over (discrete configurations) x (continuous box): see the module docstring."""

    n_sobol: int = 1024       # shared continuous points of the first sweep
    n_seeds: int = 64         # best (configuration, point) pairs that are refined
    n_local: int = 128        # points per seed and refinement round
    n_rounds: int = 6         # box half-width = 0.25 * range * 0.5^round
    max_rows: int = 4_000_000  # rows per sweep (the first sweep subsamples the continuous set to stay below)

    def best_point(self, scorer, disc: torch.Tensor, c_lo: torch.Tensor, c_hi: torch.Tensor, seed: int):
        """(row of [discrete | continuous] fp32, value) maximising ``scorer.score`` over disc x [c_lo, c_hi]."""
        dev = disc.device
        nc, dc = disc.shape[0], c_lo.shape[0]
        n0 = max(16, min(self.n_sobol, self.max_rows // max(nc, 1)))
        eng = torch.quasirandom.SobolEngine(dimension=dc, scramble=True, seed=seed)
        u = eng.draw(n0).to(dev, torch.float32)
        pts = c_lo + u * (c_hi - c_lo)
        rows = torch.cat([disc.repeat_interleave(n0, dim=0), pts.repeat(nc, 1)], dim=1)
        val = scorer.score(rows)
        k = min(self.n_seeds, rows.shape[0])
        top_v, top_i = torch.topk(val, k)
        seeds, seed_v = rows[top_i].clone(), top_v.clone()
        width = 0.25 * (c_hi - c_lo)
        for r in range(self.n_rounds):
            eng = torch.quasirandom.SobolEngine(dimension=dc, scramble=True, seed=seed + 1 + r)
            u = eng.draw(self.n_local).to(dev, torch.float32) * 2.0 - 1.0  # (n_local, dc) in [-1, 1]
            cand_c = seeds[:, None, -dc:] + u[None] * width  # (k, n_local, dc)
            cand_c = torch.minimum(torch.maximum(cand_c, c_lo), c_hi)
            cand = torch.cat([seeds[:, None, :-dc].expand(-1, self.n_local, -1), cand_c], dim=2).reshape(-1, seeds.shape[1])
            v = scorer.score(cand.contiguous()).reshape(k, self.n_local)
            bv, bi = v.max(dim=1)
            better = bv > seed_v
            pick = cand.reshape(k, self.n_local, -1)[torch.arange(k, device=dev), bi]
            seeds = torch.where(better[:, None], pick, seeds)
            seed_v = torch.where(better, bv, seed_v)
            width = width * 0.5
        j = int(torch.argmax(seed_v))
        return seeds[j], float(seed_v[j])


def recommend_hybrid(gp: DeviceGP, acq: AcqConfig, disc_comp: np.ndarray, cont_bounds: np.ndarray, batch_size: int,
                     pending: np.ndarray | None = None, n_samples: int = 512, seed: int = 0,
                     search: HybridSearch | None = None):
    """Sequential-greedy batch over a hybrid space (``optimize_acqf_mixed`` semantics, hybrid.py:110-135): returns
    (points [batch_size, d_disc + d_cont] float64 in comp-rep column order, discrete-configuration indices, joint qNEI
    value of the batch together with the initial pending points).

    ``disc_comp``: (n_configs, d_disc) comp-rep rows of the discrete subspace (it comes first in BayBE's hybrid
    comp-rep, hybrid.py:45-46); ``cont_bounds``: (2, d_cont)."""
    if acq.kind != "qNEI":
        raise NotImplementedError("the device hybrid recommender evaluates the noisy-EI family (qNEI)")
    search = search or HybridSearch()
    dev = gp.device
    disc = torch.as_tensor(np.asarray(disc_comp, dtype=np.float32), device=dev)
    cb = torch.as_tensor(np.asarray(cont_bounds, dtype=np.float32), device=dev)
    scorer = NeiScorer(gp, acq, n_samples, seed)
    pend = np.empty((0, gp.d)) if pending is None else np.asarray(pending, dtype=np.float64).reshape(-1, gp.d)
    chosen, idx = [], []
    value = 0.0
    for j in range(batch_size):
        scorer.set_pending(np.vstack([pend] + chosen) if chosen else pend)
        row, gain = search.best_point(scorer, disc, cb[0], cb[1], seed * 7919 + 31 * j)
        value = scorer.const + gain
        r64 = row.double().cpu().numpy()
        # the discrete part is one of the given rows exactly: report which
        dd = disc.shape[1]
        k = int(torch.argmin((disc - row[:dd]).abs().sum(-1)))
        r64[:dd] = np.asarray(disc_comp, dtype=np.float64)[k]
        chosen.append(r64[None])
        idx.append(k)
    return np.vstack(chosen), idx, value
