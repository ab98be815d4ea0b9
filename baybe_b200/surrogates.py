"""``GaussianProcessSurrogate`` with the reference's public surface
(``/root/reference/baybe/surrogates/base.py:49-78,213-247,308-465`` and
``gaussian_process/core.py:125-341``): ``fit(searchspace, objective, measurements)`` is cached on
its context, ``posterior`` / ``posterior_stats`` take candidates in experimental representation,
and the model owns input Normalize / output Standardize (core.py:130-141 "Scaling Workaround").

The fitted model lives on the GPU as a ``DeviceGP`` (caches built by ``bb_model_build``); every
posterior evaluation runs the wgmma kernel.  Hyper-parameter fitting (SURVEY.md row f1, *before*
the hot path) evaluates the fit criterion -- exact marginal likelihood, or the leave-one-out pseudo-likelihood
for transfer-learning search spaces -- and its gradient on the GPU (``bb_fit_eval[_loo]``, float64)
under scipy's L-BFGS-B on the BayBE preset's MAP objective
(``presets/baybe.py:57-144``: Matern-5/2 ARD, Gamma(3, rate(d)) lengthscale prior with lower bound
2.5e-2, Gamma(2, e^5) noise prior with floor 1e-4, constant mean, no output scale).
"""

from __future__ import annotations

import math
from typing import ClassVar, Sequence

import numpy as np
import pandas as pd
import torch
from attrs import define, field

from baybe_b200.engine import DeviceGP
from baybe_b200.searchspace import objective_affine

__all__ = ["GaussianProcessSurrogate", "ModelNotTrainedError", "fit_map", "fit_map_hyperparameters_device",
           "DeviceMLL", "default_fit_criterion"]

MIN_INFERRED_NOISE_LEVEL = 1e-4
MIN_LENGTHSCALE = 2.5e-2


class ModelNotTrainedError(Exception):
    """Same name/meaning as baybe.exceptions.ModelNotTrainedError (surrogates/base.py:240-243)."""


def default_fit_criterion(n_tasks: int) -> str:
    """``BayBEFitCriterionFactory`` / ``_MLLForNonTLFitCriterionFactory`` (presets/baybe.py:270-281,
    components/fit_criterion.py:61-80): exact marginal likelihood without a task parameter, the leave-one-out
    pseudo-likelihood for transfer-learning search spaces."""
    return "mll" if n_tasks <= 1 else "loo"


class DeviceMLL:
    """Fit criterion and its gradient on the GPU (``bb_fit_setup`` / ``bb_fit_eval`` / ``bb_fit_eval_loo``,
    float64): theta = [lengthscale[d] | noise | mean constant | B[T*T]].  ``criterion``: "mll" = exact marginal
    log likelihood (gpytorch ExactMarginalLogLikelihood), "loo" = leave-one-out pseudo-likelihood
    (gpytorch LeaveOneOutPseudoLikelihood); both un-normalised (the caller divides by n like gpytorch)."""

    def __init__(self, Xa: np.ndarray, y_std: np.ndarray, task_ids=None, n_tasks: int = 1,
                 family: str = "matern52", device=None, criterion: str = "mll"):
        if criterion not in ("mll", "loo"):
            raise ValueError(f"unknown fit criterion {criterion!r}")
        self.criterion = criterion
        import ctypes as C

        from baybe_b200 import _lib
        from baybe_b200.engine import _require_cuda, _stream_ptr

        self._C, self._lib_mod, self._stream_ptr = C, _lib, _stream_ptr
        self.device = _require_cuda(device)
        self.lib = _lib.load()
        self.n, self.d = Xa.shape
        self.T = int(n_tasks)
        self.family = _lib.KERNEL_FAMILY[family]
        self.np = self.d + 2 + self.T * self.T
        xa = np.ascontiguousarray(Xa, dtype=np.float64)
        yy = np.ascontiguousarray(y_std, dtype=np.float64)
        tt = None if task_ids is None else np.ascontiguousarray(task_ids, dtype=np.int32)
        nbytes = self.lib.bb_fit_workspace_bytes(self.n, self.d, self.T)
        with torch.cuda.device(self.device):
            self._ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=self.device)
            self._base = (self._ws.data_ptr() + 255) // 256 * 256
            dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
            _lib.check(self.lib.bb_fit_setup(
                C.c_void_p(self._base), nbytes, self.n, self.d, self.T, dp(xa), dp(yy),
                None if tt is None else tt.ctypes.data_as(C.POINTER(C.c_int32)), _stream_ptr()), "bb_fit_setup")

    def __call__(self, theta: np.ndarray) -> tuple[float, np.ndarray, bool]:
        """(mll, d mll / d theta, positive_definite)."""
        C = self._C
        th = np.ascontiguousarray(theta, dtype=np.float64)
        if th.shape != (self.np,):
            raise ValueError(f"theta must have {self.np} entries")
        val = C.c_double(0.0)
        grad = np.zeros(self.np)
        bad = C.c_int32(0)
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
        with torch.cuda.device(self.device):
            fn = self.lib.bb_fit_eval_loo if self.criterion == "loo" else self.lib.bb_fit_eval
            self._lib_mod.check(fn(
                C.c_void_p(self._base), self.n, self.d, self.T, self.family, dp(th), C.byref(val), dp(grad),
                C.byref(bad), self._stream_ptr()), "bb_fit_eval")
        return float(val.value), grad, bad.value == 0


def fit_map(Xn: np.ndarray, y_std: np.ndarray, active: Sequence[int], task_ids=None, n_tasks: int = 1,
            max_iter: int = 200, config=None, device=None, criterion: str | None = None,
            mll_factory=None) -> dict:
    """MAP fit of (lengthscales, noise, constant mean[, output scale][, task covariance]) on normalised inputs
    and standardised targets: maximises (log marginal likelihood + log priors) / n like
    ``botorch.fit.fit_gpytorch_mll`` on an ``ExactMarginalLogLikelihood`` (core.py:340-341), starting from the
    preset's initial values (prior modes for the BayBE preset, presets/baybe.py:100-107,134-144).  With a task
    parameter the criterion is the leave-one-out pseudo-likelihood (``default_fit_criterion``), as in the reference.

    The criterion and its gradient are evaluated on the GPU (``DeviceMLL``); priors, bounds and scipy's L-BFGS-B
    step are host code.  ``mll_factory`` lets the tests inject their float64 autograd twin of the evaluator
    (``tests/helpers.py::HostMLL``); the product never constructs a CPU evaluator."""
    from scipy.optimize import minimize

    from baybe_b200.kernels import gp_preset

    Xa = np.ascontiguousarray(np.asarray(Xn, dtype=np.float64)[:, list(active)])
    n, da = Xa.shape
    cfg = gp_preset("BAYBE", da) if config is None else config
    has_tasks = task_ids is not None
    T = n_tasks if has_tasks else 1
    crit = criterion or default_fit_criterion(T)
    mll = (mll_factory or DeviceMLL)(Xa, y_std, task_ids, T, cfg.family, device, crit)
    fit_os = cfg.outputscale and cfg.outputscale_trainable
    i_os = da + 2 if fit_os else None
    i_w = da + 2 + (1 if fit_os else 0)
    n_task_par = T * T + T if has_tasks else 0
    x0 = np.concatenate([
        np.full(da, max(cfg.lengthscale_initial_value, cfg.lengthscale_lower)),
        [max(cfg.noise_initial_value, cfg.noise_lower)], [0.0],
        [cfg.outputscale_initial_value] if fit_os else [],
        np.concatenate([np.eye(T).reshape(-1) * 0.8 + 0.2, np.full(T, 0.1)]) if n_task_par else []])
    bounds = [(cfg.lengthscale_lower, None)] * da + [(cfg.noise_lower, None), (None, None)] + \
             ([(1e-6, None)] if fit_os else []) + [(1e-6, None)] * n_task_par
    os_fixed = cfg.outputscale_initial_value if (cfg.outputscale and not fit_os) else 1.0

    def parts(x):
        osv = x[i_os] if fit_os else os_fixed
        if not n_task_par:
            return osv, np.ones((1, 1)), None
        W = x[i_w: i_w + T * T].reshape(T, T)
        v = x[i_w + T * T:]
        return osv, W @ W.T + np.diag(v), W

    def objective(x):
        osv, Bi, W = parts(x)
        theta = np.concatenate([x[: da + 2], (osv * Bi).reshape(-1)])
        val, g, ok = mll(theta)
        if not ok or not np.isfinite(val):
            return 1e10, np.zeros_like(x)
        ls, nz = x[:da], x[da]
        grad = np.zeros_like(x)
        grad[: da + 2] = g[: da + 2]
        lp = 0.0
        if cfg.lengthscale_prior is not None:
            lp += float(np.sum(cfg.lengthscale_prior.log_prob(ls)))
            grad[:da] += cfg.lengthscale_prior.grad(ls)
        if cfg.noise_prior is not None:
            lp += float(cfg.noise_prior.log_prob(nz))
            grad[da] += float(cfg.noise_prior.grad(nz))
        gB = g[da + 2:].reshape(T, T)
        if fit_os:
            grad[i_os] = float(np.sum(gB * Bi))
            if cfg.outputscale_prior is not None:
                lp += float(cfg.outputscale_prior.log_prob(osv))
                grad[i_os] += float(cfg.outputscale_prior.grad(osv))
        if n_task_par:
            grad[i_w: i_w + T * T] = (osv * (gB + gB.T) @ W).reshape(-1)
            grad[i_w + T * T:] = osv * np.diag(gB)
        return -(val + lp) / n, -grad / n

    res = minimize(objective, x0, jac=True, method="L-BFGS-B", bounds=bounds,
                   options={"maxiter": max_iter, "ftol": 1e-10, "gtol": 1e-7})
    osv, Bi, _ = parts(res.x)
    return {"lengthscale": res.x[:da].copy(), "noise": float(res.x[da]), "mean_const": float(res.x[da + 1]),
            "outputscale": float(osv) if cfg.outputscale else None,
            "task_covar": Bi if n_task_par else None, "family": cfg.family, "objective": float(res.fun),
            "n_iter": int(res.nit), "n_eval": int(res.nfev), "criterion": crit}


def fit_map_hyperparameters_device(Xn, y_std, active, task_ids=None, n_tasks: int = 1, max_iter: int = 200,
                                   device=None, config=None) -> dict:
    """``fit_map`` (kept under its round-1 name)."""
    return fit_map(Xn, y_std, active, task_ids, n_tasks, max_iter, config, device=device)


class _Posterior:
    """Marginal (t-batch) posterior with the attribute names BayBE reads from BoTorch posteriors
    (``mean``, ``variance``, ``quantile``; surrogates/base.py:352-375)."""

    def __init__(self, mean: torch.Tensor, variance: torch.Tensor):
        self.mean = mean.reshape(-1, 1, 1)
        self.variance = variance.reshape(-1, 1, 1)

    def quantile(self, value: torch.Tensor) -> torch.Tensor:
        p = torch.as_tensor(value, dtype=torch.float64, device=self.mean.device)
        z = math.sqrt(2.0) * torch.erfinv(2.0 * p - 1.0)
        return self.mean + self.variance.sqrt() * z.to(self.mean.dtype)


class _JointPosterior:
    """Joint posterior of one q-batch: ``mean`` (1, q, 1), ``variance`` (1, q, 1), ``covariance`` (q, q) -- the
    attributes BayBE reads from ``GPyTorchPosterior`` (``mean``, ``variance``, ``mvn.covariance_matrix``)."""

    def __init__(self, mean: torch.Tensor, cov: torch.Tensor):
        q = mean.numel()
        self.mean = mean.reshape(1, q, 1)
        self.covariance = cov.reshape(q, q)
        self.variance = torch.diagonal(self.covariance).reshape(1, q, 1)

    @property
    def mvn(self):
        return torch.distributions.MultivariateNormal(
            self.mean.reshape(-1).double().cpu(),
            covariance_matrix=self.covariance.double().cpu() + 1e-9 * torch.eye(self.covariance.shape[0], dtype=torch.float64))


def default_preset_name(searchspace) -> str:
    """The reference's default dispatches on search-space content (``presets/baybe.py:151-197``, ``_dispatch``): a
    ``SubstanceParameter`` anywhere in the space switches kernel, mean and likelihood to the Chen preset
    (``presets/chen.py:35-61``); every other space gets the custom-scaled BayBE preset."""
    has_substance = any(type(p_).__name__ == "SubstanceParameter" for p_ in getattr(searchspace, "parameters", ()))
    return "CHEN" if has_substance else "BAYBE"


@define
class GaussianProcessSurrogate:
    """GP surrogate whose posterior runs on the B200 engine."""

    supports_transfer_learning: ClassVar[bool] = True
    supports_multi_output: ClassVar[bool] = False

    hyperparameters: dict | None = field(default=None)
    """Optional fixed hyper-parameters {lengthscale (per active column), noise, mean_const,
    [outputscale], [task_covar], [family]}; when omitted they are MAP-fitted (BayBE preset)."""

    device: str | None = field(default=None)
    max_fit_iter: int = field(default=200)
    kernel_or_factory: object = field(default=None)
    """None (BayBE preset), a preset name ("BAYBE", "CHEN", "EDBO") or a ``baybe_b200.kernels`` kernel object
    (``GaussianProcessSurrogate(kernel_or_factory=...)``, surrogates/gaussian_process/core.py:147-186)."""

    fit_criterion: str | None = field(default=None)
    """None: the reference's default (exact MLL; leave-one-out pseudo-likelihood with a task parameter), or
    "mll" / "loo" explicitly (``GaussianProcessSurrogate(fit_criterion_or_factory=...)``, core.py:188-200)."""

    device_gp: DeviceGP | None = field(init=False, default=None, eq=False, repr=False)
    fitted_hyperparameters: dict | None = field(init=False, default=None, eq=False, repr=False)
    _searchspace = field(init=False, default=None, eq=False, repr=False)
    _objective = field(init=False, default=None, eq=False, repr=False)
    _measurements_hash: int | None = field(init=False, default=None, eq=False, repr=False)
    _target_name: str | None = field(init=False, default=None, eq=False, repr=False)

    # ---- SurrogateProtocol -------------------------------------------------------------
    def fit(self, searchspace, objective, measurements: pd.DataFrame) -> None:
        """Train on the given context; repeated calls with an unchanged context are no-ops
        (surrogates/base.py:419-424)."""
        h = int(pd.util.hash_pandas_object(measurements, index=True).sum())
        if (self.device_gp is not None and searchspace is self._searchspace
                and objective == self._objective and h == self._measurements_hash):
            return
        if getattr(objective, "is_multi_output", False):
            raise NotImplementedError("multi-output objectives are outside the B200 engine's scope")
        _, _, target = objective_affine(objective)
        if measurements[target].isna().any():
            raise ValueError("partial measurements are not supported (handle_missing_values)")
        comp = searchspace.transform(measurements, allow_extra=True)
        train_x = comp.to_numpy(dtype=np.float64)
        train_y = measurements[target].to_numpy(dtype=np.float64)
        bounds = np.asarray(searchspace.scaling_bounds.to_numpy(copy=True), dtype=np.float64)
        d = train_x.shape[1]
        task_col = searchspace.task_idx
        n_tasks = searchspace.n_tasks if task_col is not None else 1
        active = [j for j in range(d) if j != task_col]
        hp = dict(self.hyperparameters) if self.hyperparameters is not None else None
        if hp is None:
            rng = np.where(np.abs(bounds[1] - bounds[0]) < 1e-8, 1.0, bounds[1] - bounds[0])
            Xn = (train_x - bounds[0]) / rng
            ys = train_y.std(ddof=1) if len(train_y) > 1 else 1.0
            ys = ys if ys >= 1e-8 else 1.0
            tids = None if task_col is None else np.rint(train_x[:, task_col]).astype(int)
            from baybe_b200.kernels import Kernel, gp_preset, resolve_kernel

            kf = self.kernel_or_factory
            if kf is None:
                config = gp_preset(default_preset_name(searchspace), len(active))
            elif isinstance(kf, str):
                config = gp_preset(kf, len(active))
            elif isinstance(kf, Kernel):
                config = resolve_kernel(kf)
            else:
                raise TypeError("kernel_or_factory must be None, a preset name or a baybe_b200.kernels.Kernel")
            hp = fit_map(Xn, (train_y - train_y.mean()) / ys, active, tids, n_tasks, self.max_fit_iter, config,
                         device=self.device, criterion=self.fit_criterion)
        ls_full = np.full(d, -1.0)
        ls_full[active] = np.broadcast_to(np.asarray(hp["lengthscale"], dtype=np.float64), (len(active),))
        task_covar = hp.get("task_covar")
        if task_col is not None and task_covar is None:
            task_covar = np.eye(n_tasks)
        if self.device_gp is not None:
            self.device_gp.close()
        self.device_gp = DeviceGP(
            train_x, train_y, np.stack([bounds[0], bounds[1]]), hp.get("family", "matern52"), ls_full,
            hp["noise"], hp.get("mean_const", 0.0), hp.get("outputscale"), task_col, task_covar,
            device=self.device,
        )
        self.fitted_hyperparameters = hp
        self._searchspace, self._objective = searchspace, objective
        self._measurements_hash, self._target_name = h, target

    def to_botorch(self):
        raise ImportError(
            "GaussianProcessSurrogate of baybe_b200 is not backed by a botorch.models.Model; use "
            "baybe_b200.recommenders.B200Recommender, which scores through the CUDA engine")

    # ---- posterior ---------------------------------------------------------------------
    def _require_fit(self):
        if self.device_gp is None or self._searchspace is None:
            raise ModelNotTrainedError("The surrogate must be trained before a posterior can be computed.")

    def posterior(self, candidates: pd.DataFrame, *, joint: bool = False):
        """Posterior at candidates given in experimental representation (surrogates/base.py:213-247).
        ``joint=False``: marginal posteriors of all rows (t-batch; the scoring path).  ``joint=True``: ONE q-batch
        posterior with the full (q, q) covariance, computed in float64 on the device (``bb_pending_stats``, the
        routine that conditions sequential-greedy rounds on their pending points) for q <= 31."""
        self._require_fit()
        comp = self._searchspace.transform(candidates, allow_extra=True)
        if joint:
            from baybe_b200._lib import MAX_PENDING

            if len(comp) > MAX_PENDING:
                raise NotImplementedError(f"joint posteriors are implemented for q <= {MAX_PENDING} points "
                                          f"(got {len(comp)}); use joint=False for marginals of a large set")
            _, _, mean, cov = self.device_gp.pending_stats(comp.to_numpy(dtype=np.float64, copy=True))
            return _JointPosterior(mean, cov)
        return self._posterior_comp(torch.from_numpy(comp.to_numpy(dtype=np.float64, copy=True)))

    def _posterior_comp(self, candidates_comp: torch.Tensor) -> _Posterior:
        """Posterior for un-scaled comp-rep rows (surrogates/base.py:249-272)."""
        self._require_fit()
        mu, var = self.device_gp.posterior(candidates_comp)
        return _Posterior(mu, var)

    def posterior_stats(self, candidates: pd.DataFrame, stats: Sequence = ("mean", "std")) -> pd.DataFrame:
        """Posterior statistics per candidate, columns ``{target}_{stat}`` (base.py:308-384)."""
        self._require_fit()
        for st in (x for x in stats if isinstance(x, float)):
            if not 0.0 < st < 1.0:
                raise ValueError(
                    f"Posterior quantile statistics can only be computed for quantiles between 0 and 1 "
                    f"(non-inclusive). Provided value: '{st}' as part of '{stats=}'.")
        post = self.posterior(candidates, joint=False)
        out = pd.DataFrame(index=candidates.index)
        for st in stats:
            if isinstance(st, float):
                name, vals = f"Q_{st}", post.quantile(torch.tensor(st))
            elif st == "mean":
                name, vals = st, post.mean
            elif st in ("std", "var"):
                name, vals = st, post.variance
                if st == "std":
                    vals = torch.sqrt(vals)
            else:
                raise TypeError(f"The utilized posterior does not support the statistic '{st}'.")
            out[f"{self._target_name}_{name}"] = vals.reshape(-1).double().cpu().numpy()
        return out
