"""Float64 references, stated per-row error bounds and a float32 restatement of the single-target acquisition
epilogue (csrc/acq_math.cuh, the k_fused epilogue, k_acq_moments).  Test infrastructure only.

Notation: u = 2^-24 is the fp32 unit roundoff, gamma_n = n u / (1 - n u) bounds an n-step fp32 recursive sum
relative to the sum of the absolute terms.  fp32 inputs are the exact (mu, var) and base samples the kernel
consumed; the spec fields are the fp32 values of ``bb_acq_spec``.

Bound of one Monte-Carlo row (no outlier allowance):
  coef   The kernel rounds c0 = (fma(a, mu, b) - best_f) / tau and c1 = a sqrt(var) / tau:
           |dc0| <= u (|mo| + |mo - best_f|) / tau + 2 u |c0|,   |dc1| <= 4 u |c1|
         (fma, subtraction, the product and the rounded 1/tau; sqrt, two products, 1/tau).  The float64 value is
         evaluated at the four corners (c0 +- dc0, c1 (1 +- dc1)); the largest change from the centre is the term.
  terms  At the rounded coefficients each sample term is evaluated with t = fma(c1, z, c0) (|dt| <= u |t|):
           qLogEI  relu(t) + [|t| < 30] log1pf(ex2.approx(-log2e |t|)) + 0.1 rcp.approx(fma(t, t, 1))
                   relu: u |t|; tail e = exp(-|t|): (3 |t| + 8) u e (the rounded exponent, ex2.approx 2 ulp,
                   log1pf 1 ulp); 0.1/(1+t^2) = 0.1 r: 0.5 u r (dt moves r by <= 2 u r, fma 1 ulp, rcp.approx
                   2^-23); the tail skipped at |t| >= 30 counts in full, and so does a 0.1 r that rcp.approx.ftz
                   flushes to zero (|t| >= 2^63).
           qEI     relu(t): u |t|.
           qPI     rcp.approx(1 + ex2.approx(-log2e t)) = sigma: sigma (1 - sigma)(3 |t| + 4) u + 3 u sigma, and
                   sigma itself where t < -87 (ex2 overflows, rcp gives 0).
  sum    gamma_n sum_s |term_s|, n the length of the kernel's longest chain plus its tree:
           k_acq_moments  2 ceil(S/32) + 5 (lane chains of <= 32 samples, two adds each, xor tree)
           k_fused        S/2 + 8 (mc_partial: two shares of S/2, split chains; the table and exact-warp rows
                          have shorter chains)
  table  Rows whose (s0, s1) come from the tabulated tail (k_fused qLogEI, 64 <= S <= 512, S % 64 == 0): the
         interpolation error the table's comment claims (1e-5 relative) plus its construction (S/2 + 64) u, on
         the tail's share 0.1 sum_{zeta < zeta_(16)} 1/(c0 + |c1| zeta)^2, plus that share times 2^-20 for the
         1/t^2 form (t <= -1024).  The term is added to every row of a table launch: a row on the border of
         the envelope may take either path.
  output qLogEI  log(tau) + log((s0 + 0.1 s1)/S): 4 u (0.1f, product, sum, quotient) on the argument, 1 ulp of
                 each logf, 1 ulp of the sum.   qEI/qPI  s0 / S: 1 ulp.
  The arithmetic terms are divided by the row's sum (qLogEI, whose value is a log) or by S.
  qSR    fmaf(so, zbar, mo): u |mo| + 2 u |so zbar| + |so| (gamma_37 sum|z| / S + u |zbar|) + 1 ulp.
  qUCB   qSR's terms plus 1 ulp of the inner fma, c |so| zdev (5.5 u) + c |so| (dzbar + (gamma_37 + 2 u) zdev),
         c = sqrt(beta pi / 2),
         zdev = mean_s |z_s - zbar| (the lane sums of S/32 <= 32 samples and a five-level tree; both kernels).

Analytic kinds: the kernels evaluate the closed forms in float64 and round once, so the bound is 2 ulp of the
float64 value plus the smallest subnormal (EI underflows to zero or to subnormals in the far tail).
"""
from __future__ import annotations

import math

import numpy as np
import torch

import oracle
from oracle import reference_path as rp

U = 2.0**-24
F32 = np.float32
KMC_NT, KMC_K, KMC_J = 512, 16, 8
# regime classes of a qLogEI row of a table launch (mc_row_fast's envelope)
FAST, FAST_CORR, FALLBACK_T9, FALLBACK_T17, TABLE_OFF = "fast", "fast_tmin_lt_30", "fallback_t9", "fallback_t17", \
    "table_off"
CLASSES = (FAST, FAST_CORR, FALLBACK_T9, FALLBACK_T17, TABLE_OFF)
TABLE_REL = 1e-5  # interpolation error the table's comment in acq_math.cuh claims


def gamma(n: int) -> float:
    return n * U / (1.0 - n * U)


def table_applicable(kind: str, S: int) -> bool:
    return kind == "qLogEI" and 64 <= S <= 512 and S % 64 == 0


def spec32(acq) -> dict:
    """The fp32 fields of bb_acq_spec as python floats."""
    return {k: float(F32(getattr(acq, k))) for k in ("best_f", "beta", "obj_scale", "obj_shift", "tau_relu",
                                                    "tau_max", "tau_pi")}


def oracle_spec(acq) -> oracle.AcqSpec:
    """The oracle's spec with the fp32 field values the kernel sees."""
    p = spec32(acq)
    return oracle.AcqSpec(kind=acq.kind, best_f=p["best_f"], beta=p["beta"], obj_scale=p["obj_scale"],
                          obj_shift=p["obj_shift"], maximize=acq.maximize, tau_relu=p["tau_relu"],
                          tau_max=p["tau_max"], tau_pi=p["tau_pi"])


def _inv_tau(acq) -> float:
    p = spec32(acq)
    if acq.kind == "qLogEI":
        return 1.0 / p["tau_relu"]
    if acq.kind == "qPI":
        return 1.0 / p["tau_pi"]
    return 1.0


# --------------------------------------------------------------------------------------------------------------
# float32 restatement (classification and the CPU model of the table path)
# --------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 fma of fp32 operands: the product is exact in float64; one float64 rounding of the sum precedes the
    fp32 rounding (a double rounding that can differ from the device in the last bit, rarely)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def coefs32(acq, mu, var):
    """(c0, c1) as mc_coef forms them in fp32."""
    p = spec32(acq)
    mu = np.asarray(mu, F32)
    var = np.asarray(var, F32)
    mo = fma32(F32(p["obj_scale"]), mu, F32(p["obj_shift"]))
    so = F32(p["obj_scale"]) * np.sqrt(var)
    inv = F32(1.0) / F32(p["tau_relu"] if acq.kind == "qLogEI" else p["tau_pi"]) \
        if acq.kind in ("qLogEI", "qPI") else F32(1.0)
    c0 = (mo - F32(p["best_f"])) * inv
    c1 = so * inv
    return c0.astype(F32), c1.astype(F32)


def table_head(z, sgn: float) -> tuple[np.ndarray, bool]:
    """The sixteen largest zeta = sgn z (descending) and the table's validity flag (no tie at the 16th)."""
    zeta = (F32(sgn) * np.asarray(z, F32)).astype(F32)
    top = np.sort(zeta)[::-1][:KMC_K].copy()
    ok = int((zeta >= top[KMC_K - 1]).sum()) == KMC_K
    return top, ok


def table32(z, sgn: float, w0_index: int = KMC_J, tail_test_on_difference: bool = False) -> np.ndarray:
    """F[0..512] of the table in fp32 (exact reciprocals, a sequential sum).  The tail is zeta < zeta_(16), as
    the kernels test it; tail_test_on_difference restates the earlier test zeta - w < zeta_(16) - w (both
    rounded), and w0_index moves the node origin, for the planted-deviation checks."""
    zeta = (F32(sgn) * np.asarray(z, F32)).astype(F32)
    top, _ = table_head(z, sgn)
    thr, w0 = top[KMC_K - 1], top[w0_index]
    F = np.empty(KMC_NT + 1, F32)
    F[0] = F32(zeta.size - KMC_K)
    for j in range(1, KMC_NT + 1):
        a = F32(KMC_NT) / F32(j)
        w = (w0 - F32(1.0)) + a
        d = (zeta - w).astype(F32)
        keep = d < F32(thr - w) if tail_test_on_difference else zeta < thr
        d = d[keep]
        r = (F32(1.0) / (d * d)).astype(F32)
        F[j] = F32(np.cumsum(r, dtype=F32)[-1] if r.size else F32(0)) * a * a
    return F


def row_fast32(F, top, c0, c1, interpolate: bool = True, tmin_correction: bool = True):
    """mc_row_fast in fp32 for rows inside the envelope: (s0, s1).  The flags switch off parts for the
    planted-deviation checks."""
    c0 = np.asarray(c0, F32)
    ac1 = np.abs(np.asarray(c1, F32))
    t = fma32(ac1[:, None], top[None, :], c0[:, None])
    s0 = np.maximum(t, F32(0)).sum(1, dtype=F32)
    s1 = (F32(1.0) / fma32(t, t, F32(1.0))).sum(1, dtype=F32)
    if tmin_correction:
        at = np.abs(t)
        sp = np.where(at < 30, np.log1p(np.exp(-at.astype(np.float64))), 0.0).astype(F32)
        s0 = (s0 + sp.sum(1, dtype=F32)).astype(F32)
    t9 = fma32(ac1, top[KMC_J], c0)
    inv = F32(1.0) / ac1
    a = fma32(-t9, inv, F32(1.0))
    v = F32(1.0) / a
    x = v * F32(KMC_NT)
    i = np.minimum(x.astype(np.int64), KMC_NT - 1)
    fr = x - i.astype(F32)
    f0, f1 = F[i], F[i + 1]
    f = fma32(fr, f1 - f0, f0) if interpolate else f0
    q = v * inv
    s1 = fma32(f, q * q, s1)
    return s0.astype(F32), s1.astype(F32)


def classify(acq, mu, var, z) -> tuple[np.ndarray, np.ndarray]:
    """Regime of every row of a qLogEI table launch (mc_row_fast's predicate and the table's tie check, in fp32)
    and v = 1/(w - zeta_(9) + 1) for the rows inside the envelope (NaN elsewhere)."""
    sgn = -1.0 if spec32(acq)["obj_scale"] < 0 else 1.0
    top, ok = table_head(z, sgn)
    c0, c1 = coefs32(acq, mu, var)
    ac1 = np.abs(c1)
    t9 = fma32(ac1, top[KMC_J], c0)
    t17 = fma32(ac1, top[KMC_K - 1], c0)
    cls = np.empty(c0.shape, dtype=object)
    v = np.full(c0.shape, np.nan)
    if not ok:
        cls[:] = TABLE_OFF
        return cls, v
    fast = (ac1 > F32(1e-30)) & (t9 <= 0) & (t17 <= F32(-1024.0))
    tmin = np.abs(fma32(ac1[:, None], top[None, :], c0[:, None])).min(1)
    cls[:] = FALLBACK_T17
    cls[t9 > 0] = FALLBACK_T9
    cls[fast] = np.where(tmin[fast] < 30, FAST_CORR, FAST)
    with np.errstate(divide="ignore", invalid="ignore"):
        vv = F32(1.0) / fma32(-t9, F32(1.0) / ac1, F32(1.0))
    v[fast] = vv[fast]
    return cls, v


class Coverage:
    """Counts of regime classes and of the eighths of v over the rows of many launches."""

    def __init__(self):
        self.count = {c: 0 for c in CLASSES}
        self.eighths = np.zeros(8, dtype=np.int64)

    def add(self, cls, v):
        for c in CLASSES:
            self.count[c] += int((cls == c).sum())
        vv = v[np.isfinite(v)]
        np.add.at(self.eighths, np.minimum((vv * 8).astype(np.int64), 7), 1)

    def check(self, min_count: int = 1):
        """Every class and every eighth of v reached at least ``min_count`` times."""
        missing = {c: n for c, n in self.count.items() if n < min_count}
        assert not missing, f"regime classes not reached often enough: {self.count}"
        assert (self.eighths >= min_count).all(), f"eighths of v not all reached: {self.eighths.tolist()}"


# --------------------------------------------------------------------------------------------------------------
# float64 references and bounds
# --------------------------------------------------------------------------------------------------------------
def _terms64(kind: str, t: np.ndarray):
    """Per-sample terms of the MC sums at t (float64): (s0 terms, s1 terms or None)."""
    if kind == "qLogEI":
        return np.logaddexp(0.0, t), 1.0 / (1.0 + t * t)
    if kind == "qEI":
        return np.maximum(t, 0.0), None
    if kind == "qPI":
        e = np.exp(-np.abs(t))
        return np.where(t >= 0, 1.0 / (1.0 + e), e / (1.0 + e)), None
    raise ValueError(kind)


def _value_of_coefs(kind: str, acq, c0, c1, z, S: int):
    t = c0[:, None] + c1[:, None] * z[None, :]
    s0, s1 = _terms64(kind, t)
    if kind == "qLogEI":
        with np.errstate(divide="ignore"):
            return math.log(spec32(acq)["tau_relu"]) + np.log((s0.sum(1) + 0.1 * s1.sum(1)) / S)
    return s0.sum(1) / S


def mc_bound(acq, mu, var, z, path: str, table_on: bool = False, chunk: int = 2048):
    """(float64 reference [N], per-row bound [N]) of the MC kinds, for the fp32 moments (mu, var) and fp32 base
    samples z (S,) the kernel consumed.  path: "moments" (k_acq_moments) or "fused" (k_fused epilogue);
    table_on: the launch evaluated qLogEI through the table (its term is then added to every row)."""
    kind = acq.kind
    p = spec32(acq)
    mu64 = np.asarray(mu, F32).astype(np.float64)
    var64 = np.asarray(var, F32).astype(np.float64)
    z64 = np.asarray(z, F32).astype(np.float64).reshape(-1)
    S = z64.size
    ref = rp.acq_from_moments(oracle_spec(acq), torch.from_numpy(mu64), torch.from_numpy(var64),
                              torch.from_numpy(z64)).numpy()
    a, b, bf = p["obj_scale"], p["obj_shift"], p["best_f"]
    mo = a * mu64 + b
    so = a * np.sqrt(var64)
    if kind in ("qSR", "qUCB"):
        zbar = z64.mean()
        g = gamma(37)
        dzbar = g * np.abs(z64).sum() / S + U * abs(zbar)
        err = U * np.abs(mo) + 2 * U * np.abs(so * zbar) + np.abs(so) * dzbar
        if kind == "qUCB":
            c = math.sqrt(p["beta"] * math.pi / 2.0)
            zdev = np.abs(z64 - zbar).mean()
            err = err + U * np.abs(mo + so * zbar) + c * np.abs(so) * (5.5 * U * zdev + dzbar + (g + 2 * U) * zdev)
        return ref, err + U * np.abs(ref) + 1e-45
    inv = _inv_tau(acq)
    c0 = (mo - bf) * inv
    c1 = so * inv
    n = 2 * math.ceil(S / 32) + 5 if path == "moments" else S // 2 + 8
    bound = np.empty_like(ref)
    for r0 in range(0, ref.size, chunk):
        sl = slice(r0, r0 + chunk)
        cc0, cc1 = c0[sl], c1[sl]
        d0 = U * (np.abs(mo[sl]) + np.abs(mo[sl] - bf)) * inv + 2 * U * np.abs(cc0)
        centre = _value_of_coefs(kind, acq, cc0, cc1, z64, S)
        dev = np.zeros_like(centre)
        for s0_ in (-1.0, 1.0):
            for s1_ in (-1.0, 1.0):
                cv = _value_of_coefs(kind, acq, cc0 + s0_ * d0, cc1 * (1 + s1_ * 4 * U), z64, S)
                with np.errstate(invalid="ignore"):
                    dev = np.maximum(dev, np.nan_to_num(np.abs(cv - centre), nan=np.inf))
        t = cc0[:, None] + cc1[:, None] * z64[None, :]
        at = np.abs(t)
        if kind == "qLogEI":
            sp, r = _terms64(kind, t)
            e = np.exp(-at)
            tail = np.log1p(e)
            near = at < 30
            # rcp.approx.ftz flushes 1/(1+t^2) < 2^-126 (|t| >= 2^63) to zero: such a term counts in full
            term_err = (U * np.where(t > 0, at, 0.0) + np.where(near, (3 * at + 8) * U * e, tail) + 0.5 * U * r
                        + 0.1 * np.where(r < 2.0**-125, r, 0.0))
            ssum = sp.sum(1) + 0.1 * r.sum(1)
            arith = term_err.sum(1) + gamma(n) * (sp.sum(1) + 0.1 * r.sum(1))
            if table_on:
                sgn = -1.0 if a < 0 else 1.0
                zeta = sgn * z64
                thr = np.sort(zeta)[::-1][KMC_K - 1]
                tz = cc0[:, None] + np.abs(cc1)[:, None] * zeta[None, zeta < thr]
                with np.errstate(divide="ignore"):
                    tail_s1 = (1.0 / (tz * tz)).sum(1)
                arith = arith + 0.1 * tail_s1 * (TABLE_REL + (S / 2 + 64) * U + 2.0**-20)
            with np.errstate(divide="ignore", invalid="ignore"):
                rel = arith / ssum
                val = np.log(ssum / S)
                out = 4 * U + 2 * U * (np.abs(val) + abs(math.log(p["tau_relu"]))) + U * np.abs(centre)
            bound[sl] = dev + rel + out
        elif kind == "qEI":
            rl = np.maximum(t, 0.0)
            bound[sl] = dev + (U * rl.sum(1) + gamma(n) * rl.sum(1)) / S + U * np.abs(centre)
        else:  # qPI
            sg, _ = _terms64(kind, t)
            term_err = sg * (1 - sg) * (3 * at + 4) * U + 3 * U * sg + np.where(t < -87, sg, 0.0)
            bound[sl] = dev + (term_err.sum(1) + gamma(n) * sg.sum(1)) / S + U * np.abs(centre)
    return ref, bound + 1e-45


def analytic_ref(acq, mu, var) -> np.ndarray:
    """Float64 closed form on the fp32 moments and spec fields."""
    mu64 = torch.from_numpy(np.asarray(mu, F32).astype(np.float64))
    var64 = torch.from_numpy(np.asarray(var, F32).astype(np.float64))
    return rp._analytic(oracle_spec(acq), mu64, var64).numpy()


def ulp32(x) -> np.ndarray:
    x = np.abs(np.asarray(x, np.float64)).astype(F32)
    return (np.nextafter(x, F32(np.inf)) - x).astype(np.float64)


def analytic_bound(ref) -> np.ndarray:
    return 2.0 * ulp32(ref) + 2.0**-149


def worst(err, bound) -> float:
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.asarray(err, np.float64) / np.asarray(bound, np.float64)
    r = r[np.isfinite(r)]
    return float(r.max()) if r.size else 0.0


# --------------------------------------------------------------------------------------------------------------
# base-sample sets and rows placed in w = (best_f - mo) / |so|
# --------------------------------------------------------------------------------------------------------------
SAMPLE_SETS = ("sobol", "normal", "heavy", "tie16", "dup_top", "near_tie16")


def make_samples(name: str, S: int, sgn: float = 1.0, seed: int = 0) -> np.ndarray:
    """fp32 base samples (S,).  In zeta = sgn z order: "tie16" repeats the 16th largest value as the 17th (the
    table turns off), "dup_top" repeats the 3rd as the 4th (the table stays on), "near_tie16" puts the 17th one
    ulp below the 16th (the table stays on; the 17th belongs to the tail)."""
    from baybe_b200 import sobol_normal_samples

    if name == "sobol":
        return sobol_normal_samples(S, 1, seed=seed + 5)[:, 0].numpy().astype(F32)
    rng = np.random.default_rng(seed)
    if name == "heavy":
        z = rng.standard_t(2.5, size=S)
    else:
        z = rng.standard_normal(S) + 0.3  # a sample mean far from 0
    z = z.astype(F32)
    if name in ("tie16", "dup_top", "near_tie16") and S > KMC_K:
        order = np.argsort(-(F32(sgn) * z), kind="stable")
        if name == "tie16":
            z[order[16]] = z[order[15]]
        elif name == "dup_top":
            z[order[3]] = z[order[2]]
        else:
            zeta16 = F32(sgn) * z[order[15]]
            z[order[16]] = F32(sgn) * np.nextafter(zeta16, F32(-np.inf))
    return z


def rows_at(acq, sd, w) -> tuple[np.ndarray, np.ndarray]:
    """fp32 (mu, var) of rows whose objective has standard deviation |a| sd and sits at w = (best_f - mo)/|so|."""
    p = spec32(acq)
    sd = np.asarray(sd, np.float64)
    so = abs(p["obj_scale"]) * sd
    mo = p["best_f"] - np.asarray(w, np.float64) * so
    mu = (mo - p["obj_shift"]) / p["obj_scale"]
    return mu.astype(F32), (sd * sd).astype(F32)


# --------------------------------------------------------------------------------------------------------------
# joint [candidate; pending] scores (k_acq_joint)
# --------------------------------------------------------------------------------------------------------------
def kernel_jitter(attempt: int) -> float:
    """k_acq_joint's jitter of attempt 0..3, in original units (linear_operator's float32 settings)."""
    return 0.0 if attempt == 0 else float(F32(1e-6) * F32(10.0 ** (attempt - 1)))


def joint_attempt(A: np.ndarray, rule: str = "kernel"):
    """(attempt, L) of the float64 Cholesky of A + jitter I under the kernel's rule (plain, then 1e-6 10^i) or the
    oracle's (plain, then 1e-8 10^i); (None, None) when every attempt fails."""
    jits = [kernel_jitter(k) for k in range(4)] if rule == "kernel" else [0.0, 1e-8, 1e-7, 1e-6]
    for k, j in enumerate(jits):
        try:
            return k, np.linalg.cholesky(A + j * np.eye(A.shape[0]))
        except np.linalg.LinAlgError:
            continue
    return None, None


def joint_ref_and_bound(acq, mu, var, cross, pmu, pcov, z):
    """Float64 value of [candidate; pending] per row (candidate-first Cholesky with the kernel's jitter rule) and a
    bound for the Lipschitz kinds qEI, qSR, qUCB.  The fp32 Cholesky is backward stable, L L^T = A + E with
    |E| <= gamma_{Q+1} |L||L^T| (Q = 1 + P); to first order dL = L Phi(L^-1 E L^-T) (Phi: lower triangle, half the
    diagonal), so |dL| <= |L| Phi(|L^-1| |E| |L^-T|), doubled for the second-order terms.  A sample path
    y_s = m + L z_s then moves by |dL||z_s| + gamma_{Q+1} |L||z_s| + u |m|; qEI and qSR are 1-Lipschitz in every
    objective value, qUCB (1 + 2 c).  The reduction adds gamma_{S/32+6} mean_s |term| and the output 1 ulp.
    Returns (ref, bound, attempt) with attempt -1 where every attempt fails (the kernel returns NaN)."""
    p = spec32(acq)
    a, b, bf = p["obj_scale"], p["obj_shift"], p["best_f"]
    c = math.sqrt(p["beta"] * math.pi / 2.0)
    z = np.asarray(z, np.float64)
    S, Q = z.shape
    gq, gs = gamma(Q + 1), gamma(-(-S // 32) + 6)
    N = len(mu)
    ref, bound, att = np.full(N, np.nan), np.full(N, np.nan), np.full(N, -1)
    m = np.concatenate([[0.0], np.asarray(pmu, np.float64)])
    for r in range(N):
        A = np.empty((Q, Q))
        A[0, 0] = var[r]
        A[0, 1:] = A[1:, 0] = cross[r]
        A[1:, 1:] = pcov
        k, L = joint_attempt(A)
        if k is None:
            continue
        att[r] = k
        m[0] = mu[r]
        y = m[None, :] + z @ L.T
        o = a * y + b
        aL = np.abs(L)
        Li = np.abs(np.linalg.inv(L))
        M = Li @ (gq * aL @ aL.T) @ Li.T
        Phi = np.tril(M) - 0.5 * np.diag(np.diag(M))
        dL = 2.0 * aL @ Phi
        dy = np.abs(a) * (np.abs(z) @ dL.T + gq * np.abs(z) @ aL.T + U * np.abs(m)[None, :])
        if acq.kind == "qEI":
            red = np.maximum(o - bf, 0.0).max(1)
            d = dy.max(1)
        elif acq.kind == "qSR":
            red = o.max(1)
            d = dy.max(1)
        elif acq.kind == "qUCB":
            mo = o.mean(0)
            red = (mo[None, :] + c * np.abs(o - mo[None, :])).max(1)
            d = ((1 + c) * dy + (1 + c) * dy.mean(0)[None, :]).max(1)
        else:
            raise ValueError(acq.kind)
        ref[r] = red.mean()
        bound[r] = d.mean() + gs * np.abs(red).mean() + 2 * U * abs(ref[r]) + 1e-45
    return ref, bound, att
