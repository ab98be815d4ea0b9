"""Float64 oracle of the objective programs and of ``bb_objective_score`` -- test infrastructure only.

  * ``run_program``: a torch interpreter of the compiled per-target programs, written from the reference's
    ``Transformation.__call__`` formulas (transformations/basic.py, composite.py), independent of the product's numpy
    evaluator; tests/test_objectives.py checks it against the reference's own ``__call__``;
  * ``objective``: per-target programs + the desirability scalariser (desirability.py:41-70, 250-264);
  * ``objective_score_f64``: the float64 definition of ``baybe_b200::objective_score`` (same arguments), the stand-in
    engine of the CPU Campaign tests and the row-by-row reference of the GPU tests.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import oracle
from oracle.reference_path import _fatmax, _log_fatplus

OPS = {0: "AFFINE", 1: "CONST", 2: "CLAMP", 3: "TWO_SIDED", 4: "BELL", 5: "LOG", 6: "EXP", 7: "POW_INT", 8: "SIGMOID",
       9: "DUP_INPUT", 10: "ADD", 11: "MUL"}
EPS = torch.finfo(torch.float64).eps


def run_program(prog, y: torch.Tensor) -> torch.Tensor:
    """prog: [(opcode name or number, (a0, a1, a2))]; y float64."""
    y = torch.as_tensor(y, dtype=torch.float64)
    x, stack = y.clone(), []
    for op, (a0, a1, a2) in prog:
        op = OPS.get(op, op)
        if op == "AFFINE":
            x = x * a0 + a1
        elif op == "CONST":
            x = torch.full_like(x, a0)
        elif op == "CLAMP":
            x = x.clamp(None if math.isinf(a0) else a0, None if math.isinf(a1) else a1)
        elif op == "TWO_SIDED":
            x = torch.where(x < a2, (x - a2) * a0 if a0 else torch.zeros_like(x),
                            (x - a2) * a1 if a1 else torch.zeros_like(x))
        elif op == "BELL":
            x = x.sub(a0).div(a1).pow(2.0).div(2.0).neg().exp()
        elif op == "LOG":
            x = x.log()
        elif op == "EXP":
            x = x.exp()
        elif op == "POW_INT":
            x = x.pow(a0)
        elif op == "SIGMOID":
            x = 1 / (1 + torch.exp(a1 * (x - a0)))
        elif op == "DUP_INPUT":
            stack.append(x)
            x = y.clone()
        elif op == "ADD":
            x = stack.pop() + x
        elif op == "MUL":
            x = stack.pop() * x
        else:
            raise ValueError(op)
    return x


def scalarize(T: torch.Tensor, scalarizer: str, weights) -> torch.Tensor:
    w = torch.as_tensor(np.asarray(weights, dtype=np.float64), device=T.device)
    if scalarizer == "NONE":
        return T[..., 0]
    if scalarizer == "MEAN":
        return (T * w).sum(-1)
    return torch.exp(torch.sum(torch.log(T + EPS) * w, dim=-1))


def objective(programs, scalarizer: str, weights, Y: torch.Tensor) -> torch.Tensor:
    """Y [..., M] -> o [...]."""
    T = torch.stack([run_program(p, Y[..., m]) for m, p in enumerate(programs)], -1)
    return scalarize(T, scalarizer, weights)


def _programs(ops, args, n_ops):
    progs, k = [], 0
    for n in n_ops:
        progs.append([(int(ops[k + i]), tuple(args[3 * (k + i): 3 * (k + i) + 3])) for i in range(n)])
        k += n
    return progs


def candidate_samples(mu, var, cross, linv, w, z) -> torch.Tensor:
    """Y [S, N, M] of the kernel's conditional form (float64)."""
    M, N = mu.shape
    P = 0 if cross is None else cross.shape[2]
    Q = P + 1
    z = z.double()
    Y = torch.empty(z.shape[0], N, M, dtype=torch.float64)
    for m in range(M):
        zx = z[:, m * Q + P]
        if P == 0:
            Y[:, :, m] = mu[m].double()[None] + var[m].double().clamp_min(0).sqrt()[None] * zx[:, None]
        else:
            c = cross[m].double()
            r2 = (c @ linv[m].double().T).pow(2).sum(1)
            sd = (var[m].double() - r2).clamp_min(0).sqrt()
            Y[:, :, m] = mu[m].double()[None] + w[m].double() @ c.T + sd[None] * zx[:, None]
    return Y


def terms(kind: str, o: torch.Tensor, best_f: float, beta: float, tau_relu: float, tau_pi: float) -> torch.Tensor:
    """Per-sample term of every point, o [S, ...]."""
    if kind == "qLogEI":
        return _log_fatplus(o - best_f, tau_relu)
    if kind == "qEI":
        return (o - best_f).clamp_min(0.0)
    if kind == "qPI":
        return torch.sigmoid((o - best_f) / tau_pi)
    if kind == "qSR":
        return o
    m = o.mean(0, keepdim=True)
    return m + math.sqrt(beta * math.pi / 2) * (o - m).abs()


def values_from_samples(kind: str, o: torch.Tensor, pend_terms, best_f, beta, tau_relu, tau_max, tau_pi):
    """o [S, N] candidate objective samples, pend_terms [S, P] or None -> value per candidate (float64)."""
    tx = terms(kind, o, best_f, beta, tau_relu, tau_pi)
    S = o.shape[0]
    if pend_terms is None or pend_terms.shape[1] == 0:
        if kind == "qLogEI":
            return torch.logsumexp(tx, 0) - math.log(S)
        return tx.mean(0)
    pt = torch.as_tensor(pend_terms, dtype=torch.float64)
    allt = torch.cat([tx[:, :, None], pt[:, None, :].expand(-1, tx.shape[1], -1)], -1)  # (S, N, 1+P)
    if kind == "qLogEI":
        return torch.logsumexp(_fatmax(allt, tau_max, dim=-1).reshape(S, -1), 0) - math.log(S)
    return allt.amax(-1).mean(0)


def objective_score_f64(mu, var, cross, linv, w, pend_terms, z, keep, kind, params, scalarizer, ops, args, n_ops,
                        weights, index_offset, want_scores):
    """Float64 stand-in of ``baybe_b200::objective_score`` (same arguments, the definition of csrc/objective.cu)."""
    from baybe_b200 import _lib
    from baybe_b200.engine import AcqConfig, pack_best

    cfg = AcqConfig.from_params(kind, params)
    scal = {v: k for k, v in _lib.OBJ_SCALARIZER.items()}[scalarizer]
    progs = _programs(ops, args, n_ops)
    mu, var = mu.double().cpu(), var.double().cpu()
    if not cfg.is_mc:  # MEAN over affine targets: Gaussian moments
        a = torch.tensor([p[0][1][0] if p else 1.0 for p in progs], dtype=torch.float64)
        b = torch.tensor([p[0][1][1] if p else 0.0 for p in progs], dtype=torch.float64)
        wt = torch.tensor(weights, dtype=torch.float64)
        mean = ((wt * a)[:, None] * mu + (wt * b)[:, None]).sum(0)
        v = ((wt * a)[:, None] ** 2 * var).sum(0)
        acq = oracle.AcqSpec(kind=cfg.kind, best_f=cfg.best_f, beta=cfg.beta, maximize=cfg.maximize)
        val = oracle.reference_path.acq_from_moments(acq, mean, v.clamp_min(1e-300))
    else:
        Y = candidate_samples(mu, var, None if cross is None else cross.cpu(), None if linv is None else linv.cpu(),
                              None if w is None else w.cpu(), z.cpu())
        o = objective(progs, scal, weights, Y)
        val = values_from_samples(cfg.kind, o, None if pend_terms is None else pend_terms.cpu(), cfg.best_f, cfg.beta,
                                  cfg.tau_relu, cfg.tau_max, cfg.tau_pi)
    s32 = val.float()
    best = -(1 << 63)
    for i in range(len(s32)):
        if (keep is None or int(keep[i]) != 0) and not math.isnan(float(s32[i])):
            best = max(best, pack_best(float(s32[i]), i + int(index_offset)))
    return (s32 if want_scores else None), torch.tensor([best], dtype=torch.int64)
