"""Objectives that are not affine in the modelled targets, on the engine: ``DesirabilityObjective``
(``/root/reference/baybe/objectives/desirability.py``) and single targets with a non-affine transformation
(``objectives/base.py:130-150``, ``transformations/basic.py``, ``transformations/composite.py``).

The reference applies ``objective.to_botorch()`` to posterior samples of one model per target
(``acquisition/_builder.py:211-254``).  Here every oriented target's transformation is compiled into a postfix
program (``compile_objective``) that ``bb_objective_score`` (csrc/objective.cu) runs on each sample; the host keeps
what does not depend on the candidate, in float64: best_f (the objective of the posterior means at the training
inputs, ``_builder.py:141-161, 256-265``) and, with pending points, the pending points' per-sample terms
(``evaluate_program`` / ``scalarize`` are the float64 twins of the device interpreter).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from baybe_b200 import _lib
from baybe_b200.engine import AcqConfig
from baybe_b200.scoring import Scorer

__all__ = ["CompiledObjective", "compile_objective", "evaluate_program", "scalarize", "evaluate_objective",
           "uses_objective_scorer", "pending_conditioning", "ObjectiveScorer", "build_objective_scorer"]

GEOM_EPS = float(np.finfo(np.float64).eps)  # torch.finfo(float64).eps of _geometric_mean (desirability.py:63)
_OP = _lib.OBJ_OP


def _objective_score(*args):
    """``baybe_b200::objective_score`` (engine.py); a module-level seam so that CPU tests can put a float64
    stand-in here."""
    return torch.ops.baybe_b200.objective_score(*args)


class CompiledObjective:
    """Per-target programs [(opcode name, (arg0, arg1, arg2)), ...] (model order), the scalarizer
    ("NONE" / "MEAN" / "GEOM_MEAN") and the normalised weights."""

    def __init__(self, names, programs, scalarizer: str, weights):
        self.names = tuple(names)
        self.programs = [list(p) for p in programs]
        self.scalarizer = scalarizer
        self.weights = np.asarray(weights, dtype=np.float64)

    @property
    def M(self) -> int:
        return len(self.programs)

    def flat(self) -> tuple[list[int], list[float], list[int]]:
        """(opcodes, args (three per op), ops per target) -- the flattened form the custom op takes."""
        ops = [_OP[o] for p in self.programs for o, _ in p]
        args = [float(v) for p in self.programs for _, a in p for v in a]
        return ops, args, [len(p) for p in self.programs]


# ---- compiling the reference's transformations ----------------------------------------------------------------------
def _bound(v, default: float) -> float:
    return default if v is None else float(v)


def _ops(tr, prefix: list) -> list:
    """Ops that replace the top of the stack v = prefix(y) by tr(v).  The second branch of an Additive /
    Multiplicative transformation starts from DUP_INPUT (y) and re-applies the prefix, so composites nest anywhere."""
    name = type(tr).__name__
    if name == "IdentityTransformation":
        return []
    if name == "AffineTransformation":
        return [("AFFINE", (float(tr.factor), float(tr.shift), 0.0))]
    if name == "ClampingTransformation":
        return [("CLAMP", (_bound(tr.cutoffs.lower, -math.inf), _bound(tr.cutoffs.upper, math.inf), 0.0))]
    if name == "TwoSidedAffineTransformation":
        return [("TWO_SIDED", (float(tr.slope_left), float(tr.slope_right), float(tr.midpoint)))]
    if name == "BellTransformation":
        return [("BELL", (float(tr.center), float(tr.sigma), 0.0))]
    if name in ("AbsoluteTransformation", "TriangularTransformation"):
        return _ops(tr._transformation, prefix)
    if name == "LogarithmicTransformation":
        return [("LOG", (0.0, 0.0, 0.0))]
    if name == "ExponentialTransformation":
        return [("EXP", (0.0, 0.0, 0.0))]
    if name == "PowerTransformation":
        e = float(tr.exponent)
        if e != int(e):
            raise NotImplementedError(
                f"PowerTransformation(exponent={e}): non-integer powers are not supported by the B200 engine (the "
                "reference raises for any negative sample, which Gaussian posterior samples make near certain)")
        return [("POW_INT", (e, 0.0, 0.0))]
    if name == "SigmoidTransformation":
        return [("SIGMOID", (float(tr.center), float(tr.steepness), 0.0))]
    if name == "ChainedTransformation":
        out, pre = [], list(prefix)
        for t in tr.transformations:
            o = _ops(t, pre)
            out += o
            pre += o
        return out
    if name in ("AdditiveTransformation", "MultiplicativeTransformation"):
        t0, t1 = tr.transformations
        return (_ops(t0, prefix) + [("DUP_INPUT", (0.0, 0.0, 0.0))] + list(prefix) + _ops(t1, prefix)
                + [("ADD" if name.startswith("Additive") else "MUL", (0.0, 0.0, 0.0))])
    if name == "CustomTransformation":
        raise NotImplementedError("CustomTransformation wraps an arbitrary Python callable, which the B200 engine "
                                  "cannot run on the device; express the transformation with the built-in ones")
    raise NotImplementedError(f"target transformation {name} is not supported by the B200 engine")


def _fold(prog: list) -> list:
    """Join consecutive AFFINE ops; an affine map of factor 0 becomes CONST (AffineTransformation.__call__ returns
    the shift whatever the input, NaN included)."""
    out = []
    for op, a in prog:
        if op == "AFFINE" and out and out[-1][0] == "AFFINE":
            f1, s1, _ = out[-1][1]
            out[-1] = ("AFFINE", (f1 * a[0], s1 * a[0] + a[1], 0.0))
        else:
            out.append((op, tuple(a)))
    return [("CONST", (a[1], 0.0, 0.0)) if op == "AFFINE" and a[0] == 0.0 else (op, a) for op, a in out]


def _check_program(prog: list, name: str) -> None:
    if len(prog) > _lib.OBJ_MAX_OPS:
        raise NotImplementedError(f"the transformation of target '{name}' compiles to {len(prog)} ops, more than the "
                                  f"{_lib.OBJ_MAX_OPS} the B200 engine supports")
    depth = 1
    for op, _ in prog:
        depth += 1 if op == "DUP_INPUT" else -1 if op in ("ADD", "MUL") else 0
        if depth > _lib.OBJ_MAX_STACK:
            raise NotImplementedError(f"the transformation of target '{name}' nests composites deeper than the "
                                      f"evaluation stack of {_lib.OBJ_MAX_STACK} entries the B200 engine supports")


def program_of(transformation, name: str = "target") -> list:
    prog = _fold(_ops(transformation, []))
    _check_program(prog, name)
    return prog


def is_desirability(objective) -> bool:
    return type(objective).__name__ == "DesirabilityObjective"


def uses_objective_scorer(objective) -> bool:
    """True where ``bb_objective_score`` serves the objective: desirability computed on posterior samples, and single
    targets whose transformation is not affine.  Affine single targets stay on the fused path."""
    from baybe_b200.searchspace import target_affine

    if is_desirability(objective):
        return not getattr(objective, "as_pre_transformation", False)
    if getattr(objective, "is_multi_output", False):
        return False
    targets = getattr(objective, "targets", ())
    if len(targets) != 1:
        return False
    try:
        target_affine(targets[0])
    except NotImplementedError:
        return True
    return False


def compile_objective(objective, analytic: bool = False) -> CompiledObjective:
    """Programs of the reference's oriented targets (``Objective._oriented_targets``: negation for minimised single
    targets, 1 - y for minimised desirability targets).  ``analytic=True`` gives the orientation of the reference's
    posterior transform instead (desirability.py:294-320: minimised targets negated, without the + 1)."""
    targets = tuple(objective.targets)
    for t in targets:
        if type(t).__name__ != "NumericalTarget":
            raise NotImplementedError(f"target '{t.name}' of type {type(t).__name__}: only numerical targets are "
                                      "supported by the B200 engine's objective programs")
    if len(targets) > _lib.OBJ_MAX_TARGETS:
        raise NotImplementedError(f"{len(targets)} targets: the B200 engine supports objectives of at most "
                                  f"{_lib.OBJ_MAX_TARGETS} targets")
    if analytic:
        from baybe_b200.searchspace import target_affine

        programs = []
        for t in targets:
            a, b = target_affine(t)
            programs.append([("AFFINE", (a, b, 0.0))])
    else:
        programs = [program_of(t.transformation, t.name) for t in objective._oriented_targets]
    names = [t.name for t in targets]
    if is_desirability(objective):
        return CompiledObjective(names, programs, objective.scalarizer.name, objective.normalized_weights)
    return CompiledObjective(names, programs, "NONE", [1.0])


# ---- float64 evaluation (best_f, pending terms, the pre-transformed desirability) -----------------------------------
def evaluate_program(prog: list, y) -> np.ndarray:
    """The device interpreter's definition in float64."""
    y = np.asarray(y, dtype=np.float64)
    x = y.copy()
    stack: list[np.ndarray] = []
    with np.errstate(all="ignore"):
        for op, (a0, a1, a2) in prog:
            if op == "AFFINE":
                x = x * a0 + a1
            elif op == "CONST":
                x = np.full_like(x, a0)
            elif op == "CLAMP":
                x = np.where(x < a0, a0, np.where(x > a1, a1, x))
            elif op == "TWO_SIDED":
                d = x - a2
                x = np.where(x < a2, d * a0 if a0 != 0.0 else 0.0, d * a1 if a1 != 0.0 else 0.0)
            elif op == "BELL":
                x = np.exp(-(((x - a0) / a1) ** 2) / 2.0)
            elif op == "LOG":
                x = np.log(x)
            elif op == "EXP":
                x = np.exp(x)
            elif op == "POW_INT":
                x = np.power(x, a0)
            elif op == "SIGMOID":
                x = 1.0 / (1.0 + np.exp(a1 * (x - a0)))
            elif op == "DUP_INPUT":
                stack.append(x)
                x = y.copy()
            elif op == "ADD":
                x = stack.pop() + x
            elif op == "MUL":
                x = stack.pop() * x
            else:
                raise ValueError(f"unknown op {op!r}")
    return x


def scalarize(T, scalarizer: str, weights) -> np.ndarray:
    """T [..., M] -> o [...]: the single column, the weighted mean, or the weighted geometric mean with eps."""
    T = np.asarray(T, dtype=np.float64)
    w = np.asarray(weights, dtype=np.float64)
    if scalarizer == "NONE":
        return T[..., 0]
    if scalarizer == "MEAN":
        return (T * w).sum(-1)
    if scalarizer == "GEOM_MEAN":
        with np.errstate(all="ignore"):
            return np.exp((np.log(T + GEOM_EPS) * w).sum(-1))
    raise NotImplementedError(f"No scalarization mechanism defined for '{scalarizer}'.")


def evaluate_objective(comp: CompiledObjective, Y) -> np.ndarray:
    """Y [..., M] raw target values (model order) -> objective values [...]."""
    Y = np.asarray(Y, dtype=np.float64)
    T = np.stack([evaluate_program(p, Y[..., m]) for m, p in enumerate(comp.programs)], -1)
    return scalarize(T, comp.scalarizer, comp.weights)


def kind_terms(cfg: AcqConfig, o: np.ndarray) -> np.ndarray:
    """Per-sample term of every point of a q-batch, o [S, P] (the pending terms of ``bb_objective_score``)."""
    if cfg.kind == "qLogEI":
        t = (o - cfg.best_f) / cfg.tau_relu
        return math.log(cfg.tau_relu) + np.log(np.logaddexp(0.0, t) + 0.1 / (1.0 + t * t))
    if cfg.kind == "qEI":
        return np.maximum(o - cfg.best_f, 0.0)
    if cfg.kind == "qPI":
        with np.errstate(over="ignore"):  # exp overflows to inf far below best_f: the term is 0 there
            return 1.0 / (1.0 + np.exp(-(o - cfg.best_f) / cfg.tau_pi))
    if cfg.kind == "qSR":
        return o
    if cfg.kind == "qUCB":
        m = o.mean(axis=0, keepdims=True)
        return m + math.sqrt(cfg.beta * math.pi / 2.0) * np.abs(o - m)
    raise ValueError(f"{cfg.kind} has no per-sample term")


# ---- pending points (shared with baybe_b200.multiobjective.HviScorer) -----------------------------------------------
def pending_conditioning(gps, pend: np.ndarray, z: torch.Tensor):
    """Per target m of P pending points: (pending rows, beta), L_PP^-1, w_m = rows (L^-T z_{s,P})^T and the pending
    samples y_P,s = mu_P + L z_{s,P}.  z: (S, M(1+P)) float64, column m(1+P)+j = pending point j of target m.
    Returns (stats, linv [M,P,P], w [M,S,P], ys [S,P,M]), float64."""
    from baybe_b200.multiobjective import _psd_cholesky

    P, M, S = len(pend), len(gps), z.shape[0]
    Q = P + 1
    stats, linv, w = [], np.zeros((M, P, P)), np.zeros((M, S, P))
    ys = np.zeros((S, P, M))
    for m, gp in enumerate(gps):
        px, beta, pmu, pcov = gp.pending_stats(pend)
        stats.append((px, beta))
        K = pcov.double().cpu().numpy()
        L = _psd_cholesky(K)
        Linv = np.linalg.inv(L)
        linv[m] = Linv
        zp = z[:, m * Q: m * Q + P].numpy()
        w[m] = zp @ Linv  # rows: (L^-T z_s)^T
        ys[:, :, m] = pmu.double().cpu().numpy()[None, :] + zp @ L.T
    return stats, linv, w, ys


class ObjectiveScorer(Scorer):
    """MC (and, for MEAN desirability over affine targets, analytic) acquisition values of a compiled objective over
    one model per target.
    `comp` is evaluated on the samples; `analytic` (analytic kinds only) gives the Gaussian moments."""

    def __init__(self, gps, cfg: AcqConfig, comp: CompiledObjective, analytic: CompiledObjective | None = None):
        self.gps, self.cfg, self.comp = list(gps), cfg, comp
        self.M = len(self.gps)
        if self.M != comp.M:
            raise ValueError(f"{self.M} models for an objective of {comp.M} targets")
        self.device = self.gps[0].device
        self.kernel_comp = analytic if not cfg.is_mc else comp
        if self.kernel_comp is None:
            raise ValueError(f"{cfg.kind} needs the analytic (Gaussian) form of the objective")

    def values(self, x, pend: np.ndarray | None, z: torch.Tensor | None, keep=None, index_offset: int = 0,
               want_scores: bool = True):
        """(scores or None, packed best key, report) for every row of x; the kernel's value already is the value of
        the batch [x; pending], so `report` is the identity."""
        M = self.M
        P = 0 if pend is None else len(pend)
        if P and not self.cfg.is_mc:
            raise ValueError(f"{self.cfg.kind} is analytic and takes no pending points")
        xd = self.gps[0].prepare(x)
        cross = linv = w = terms = zd = None
        if z is not None:
            z = torch.as_tensor(z, dtype=torch.float64).reshape(-1, M * (1 + P))
            zd = z.to(self.device, torch.float32).contiguous()
        if P == 0:
            post = [gp.posterior(xd) for gp in self.gps]
        else:
            stats, linv_h, w_h, ys = pending_conditioning(self.gps, np.asarray(pend, dtype=np.float64), z)
            post = [gp.cross_covariance(xd, px, beta) for gp, (px, beta) in zip(self.gps, stats)]
            cross = torch.stack([c for _, _, c in post]).contiguous()
            linv = torch.from_numpy(linv_h).to(self.device, torch.float32)
            w = torch.from_numpy(w_h).to(self.device, torch.float32)
            terms = torch.from_numpy(kind_terms(self.cfg, evaluate_objective(self.comp, ys))).to(
                self.device, torch.float32).contiguous()
        mu = torch.stack([p[0] for p in post]).contiguous()
        var = torch.stack([p[1] for p in post]).contiguous()
        kc = self.kernel_comp
        ops, args, n_ops = kc.flat()
        scores, key = _objective_score(
            mu, var, cross, linv, w, terms, zd, keep, _lib.ACQ_KIND[self.cfg.kind], self.cfg.params(),
            _lib.OBJ_SCALARIZER[kc.scalarizer], ops, args, n_ops, [float(v) for v in kc.weights], int(index_offset),
            bool(want_scores))
        return (scores if want_scores else None), key, (lambda v: v)

    def n_sample_columns(self, n_other: int) -> int | None:
        """M(1+P) (the layout of ``HviScorer``); None for analytic kinds."""
        return self.M * (1 + n_other) if self.cfg.is_mc else None


def _incompatibility(msg: str) -> Exception:
    try:
        from baybe.exceptions import IncompatibilityError

        return IncompatibilityError(msg)
    except ImportError:  # pragma: no cover - baybe absent
        return ValueError(msg)


def build_objective_scorer(acqf, gps, searchspace, objective, measurements) -> ObjectiveScorer:
    """The reference's builder steps for a non-affine objective (_builder.py:141-161, 211-265) on the engine.
    `acqf`: an engine acquisition spec; `gps`: one DeviceGP per target, in target order."""
    from baybe_b200.multiobjective import _error

    kind = acqf.abbreviation
    mc = ("qLogEI", "qEI", "qPI", "qSR", "qUCB")
    analytic_kinds = ("EI", "LogEI", "PI", "UCB", "PM", "PSTD")
    if kind not in mc + analytic_kinds:
        raise _error("IncompatibleAcquisitionFunctionError")(
            f"'{type(acqf).__name__}' is not implemented by the B200 engine for objectives that are not affine in "
            f"the targets (available: {', '.join(mc + analytic_kinds)})")
    comp = compile_objective(objective)
    analytic = None
    if kind in analytic_kinds:
        if not (comp.scalarizer == "MEAN" and all(
                type(t.transformation).__name__ in ("IdentityTransformation", "AffineTransformation")
                for t in objective.targets)):
            raise _incompatibility(
                f"The selected analytical acquisition function '{type(acqf).__name__}' is incompatible with the "
                f"assigned objective '{type(objective).__name__}' because the former requires a Gaussian "
                "distribution and the latter is configured to produce non-Gaussian outcomes.")
        analytic = compile_objective(objective, analytic=True)
    kw = acqf._engine_kwargs()
    best_f = 0.0
    if kind in ("qLogEI", "qEI", "qPI", "EI", "LogEI", "PI"):
        # max over the training inputs of the full objective of the posterior means; for analytic kinds this keeps
        # the reference's + 1 of minimised desirability targets, which its posterior transform omits
        train_x = torch.from_numpy(searchspace.transform(measurements, allow_extra=True).to_numpy(dtype=np.float64))
        means = np.stack([gp.posterior(train_x)[0].double().cpu().numpy() for gp in gps], axis=1)
        best_f = float(np.max(evaluate_objective(comp, means)))
    cfg = AcqConfig(kind=kind, best_f=best_f, **kw)
    return ObjectiveScorer(gps, cfg, comp, analytic)
