"""The single-target acquisition epilogue against float64 on the exact fp32 moments it scored.

``gp.posterior(x)`` runs the same ``launch_fused`` instantiation and grid as ``gp.score`` (``has_acq`` is a run-time
flag), so it returns the fp32 (mu, var) the scoring epilogue consumed.  The premise is checked first: for every
analytic kind ``score_fused`` equals ``acq_score(posterior)`` bit for bit.  Every score is then compared with the
oracle's float64 value on those fp32 moments, ``oracle.reference_path.acq_from_moments``, within the per-row bound
derived in tests/acq_epilogue_ref.py (coefficient rounding, per-term intrinsics, the summation chains, the
qLogEI table, the output), with no outlier allowance.

qLogEI on k_fused is swept over each table builder: the in-CTA build (N <= 1024 rows, grid <= 8), the grid build
``k_mc_table_grid`` (N = 2000: 16 CTAs) and ``k_mc_table`` of a wide fingerprint model.  Every row is classified
by the fp32 restatement of mc_row_fast's envelope and the tie check; each regime and each eighth of v in [0, 1]
must be reached.  ``bb_acq_score`` (k_acq_moments) is checked on synthetic moments across its sample-count tails,
the analytic branch points and the fp32 domain edge of qLogEI; ``bb_acq_score_joint`` on candidates collinear with
a pending point, so that each of its four jitter attempts and the all-fail NaN occurs; the arg-max keys against
torch.argmax / torch.topk semantics.

The joint reference applies the kernel's jitter rule (linear_operator's float32 settings: 1e-6 10^i in original
units); the oracle's ``_chol_with_jitter`` uses the float64 settings (1e-8 10^i).  The two differ where jitter
engages: at s_y = 1e-3 the 1e-6 jitter is as large as the variances and moves L by about s_y, and at s_y = 1 the
float64 rule, which stops at 1e-6, fails on rows the kernel factors with 1e-5 or 1e-4.  The test prints both.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from baybe_b200 import AcqConfig, DeviceGP, _lib
from baybe_b200.bits import pack_bits
from baybe_b200.engine import decode_best
from baybe_b200.synthetic import fingerprint_workload, numeric_grid_workload
from tests import acq_epilogue_ref as ar

pytestmark = pytest.mark.gpu

F32 = np.float32
MC_KINDS = ["qLogEI", "qEI", "qPI", "qSR", "qUCB"]
ANALYTIC_KINDS = ["EI", "LogEI", "PI", "UCB", "PM", "PSTD"]
FUSED_S = [16, 48, 64, 128, 448, 512, 576, 1024]
SCALES = [1.0, -0.7]
SHIFT = 0.25

_MODELS = {}


def _model(name, dev):
    """(gp, candidate tensor) per table builder: "cta" in-CTA build, "grid" k_mc_table_grid, "wide" k_mc_table."""
    if name not in _MODELS:
        if name == "cta":
            w = numeric_grid_workload(N=1000, d=6, n=64, seed=11)
        elif name == "grid":
            w = numeric_grid_workload(N=2000, d=6, n=64, seed=12)
        else:
            w = fingerprint_workload(N=1000, d=2048, n=128, seed=13)
        gp = DeviceGP(device=dev, **w.gp_kwargs())
        x = torch.from_numpy(pack_bits(w.candidates) if name == "wide" else w.candidates)
        _MODELS[name] = (gp, gp.prepare(x))
    return _MODELS[name]


def _moments(gp, x):
    mu, var = gp.posterior(x)
    return mu.cpu().numpy(), var.cpu().numpy()


def _score(gp, acq, x, z):
    zt = None if z is None else torch.from_numpy(np.asarray(z, F32)).to(gp.device)
    s, key = gp.score(acq, x, zt)
    return s.cpu().numpy().astype(np.float64), key


def _acq_score(acq, mu, var, z, dev):
    zt = None if z is None else torch.from_numpy(np.asarray(z, F32)).to(dev)
    out = torch.ops.baybe_b200.acq_score(torch.from_numpy(np.asarray(mu, F32)).to(dev),
                                         torch.from_numpy(np.asarray(var, F32)).to(dev), zt,
                                         _lib.ACQ_KIND[acq.kind], acq.params())
    return out.cpu().numpy().astype(np.float64)


def _check(name, got, ref, bound):
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{name}: {int(bad.sum())} rows outside the bound, worst err/bound "
                           f"{ar.worst(err, bound):.3g}; first rows {np.nonzero(bad)[0][:5].tolist()}: got "
                           f"{got[bad][:3]}, ref {ref[bad][:3]}, bound {bound[bad][:3]}")
    return ar.worst(err, bound)


# ------------------------------------------------------------------------------------------------------------------
# k_fused epilogue
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("builder", ["cta", "grid", "wide"])
@pytest.mark.parametrize("scale", SCALES)
def test_fused_analytic_scores_equal_acq_score_of_posterior_and_float64(builder, scale, cuda_device):
    gp, x = _model(builder, cuda_device)
    mu, var = _moments(gp, x)
    mo = scale * mu.astype(np.float64) + SHIFT
    for kind in ANALYTIC_KINDS:
        acq = AcqConfig(kind=kind, best_f=float(np.quantile(mo, 0.9)), beta=0.3, obj_scale=scale, obj_shift=SHIFT)
        got, key = _score(gp, acq, x, None)
        direct = _acq_score(acq, mu, var, None, cuda_device)
        assert np.array_equal(got, direct), f"{builder} {kind}: score_fused differs from acq_score(posterior)"
        ref = ar.analytic_ref(acq, mu, var)
        r = _check(f"{builder} {kind}", got, ref, ar.analytic_bound(ref))
        assert decode_best(key)[1] == int(np.argmax(got))
        print(f"{builder} a={scale:+.1f} {kind}: worst err/bound {r:.3f}")


@pytest.mark.parametrize("builder", ["cta", "grid", "wide"])
@pytest.mark.parametrize("kind", ["qEI", "qPI", "qSR", "qUCB"])
@pytest.mark.parametrize("scale", SCALES)
def test_fused_mc_scores_within_bound(builder, kind, scale, cuda_device):
    gp, x = _model(builder, cuda_device)
    mu, var = _moments(gp, x)
    mo = scale * mu.astype(np.float64) + SHIFT
    worst = {}
    for S in FUSED_S:
        for name in ("sobol", "normal"):
            z = ar.make_samples(name, S, 1.0, seed=S)
            for q in (0.5, 0.95):
                acq = AcqConfig(kind=kind, best_f=float(np.quantile(mo, q)), beta=0.3, obj_scale=scale,
                                obj_shift=SHIFT)
                got, key = _score(gp, acq, x, z)
                ref, bound = ar.mc_bound(acq, mu, var, z, "fused")
                worst[S] = max(worst.get(S, 0.0), _check(f"{builder} {kind} S={S} {name}", got, ref, bound))
                assert decode_best(key)[1] == int(np.argmax(got))
    print(f"{builder} {kind} a={scale:+.1f}: worst err/bound per S {worst}")


def _best_f_sweep(mo, so, top, tau):
    """best_f values whose rows cover w = (best_f - mo)/|so| from zeta_(9) - 2 to zeta_(1) + 2 and far beyond, and
    rows within 30 tau of zeta_(9) (the tmin < 30 correction)."""
    targets = [top[ar.KMC_J] - 2, top[ar.KMC_J] - 0.3, top[ar.KMC_J], top[ar.KMC_J] + 0.05, top[ar.KMC_J] + 0.4,
               top[0] + 2, top[0] + 60]
    out = [float(np.median(mo + np.abs(so) * t)) for t in targets]
    for r in np.argsort(-np.abs(so))[:3]:  # t9 = -10 at the rows of largest sd
        out.append(float(mo[r] + abs(so[r]) * top[ar.KMC_J] + 10 * tau))
    return out


@pytest.mark.parametrize("builder", ["cta", "grid", "wide"])
@pytest.mark.parametrize("scale", SCALES)
def test_fused_qlogei_regimes_within_bound(builder, scale, cuda_device):
    gp, x = _model(builder, cuda_device)
    mu, var = _moments(gp, x)
    sgn = -1.0 if scale < 0 else 1.0
    mo = scale * mu.astype(np.float64) + SHIFT
    so = scale * np.sqrt(var.astype(np.float64))
    cov = ar.Coverage()
    per_class: dict = {}
    runs = [(S, "sobol") for S in FUSED_S] + [(S, n) for S in (64, 512) for n in ar.SAMPLE_SETS[1:]]
    for S, name in runs:
        z = ar.make_samples(name, S, sgn, seed=S)
        table = ar.table_applicable("qLogEI", S)
        top, ok = ar.table_head(z, sgn)
        for tau in (1e-6, 1e-3):
            fs = _best_f_sweep(mo, so, top, tau) if table else [float(np.quantile(mo, q)) for q in (0.5, 0.99)]
            for bf in fs:
                acq = AcqConfig(kind="qLogEI", best_f=bf, obj_scale=scale, obj_shift=SHIFT, tau_relu=tau)
                got, key = _score(gp, acq, x, z)
                ref, bound = ar.mc_bound(acq, mu, var, z, "fused", table_on=table and ok)
                label = f"{builder} S={S} {name} tau={tau:g} best_f={bf:.6g}"
                _check(label, got, ref, bound)
                assert decode_best(key)[1] == int(np.argmax(got)), label
                if not table:
                    continue
                cls, v = ar.classify(acq, mu, var, z)
                cov.add(cls, v)
                err = np.abs(got - ref)
                for c in ar.CLASSES:
                    m = cls == c
                    if m.any():
                        per_class[c] = max(per_class.get(c, 0.0), ar.worst(err[m], bound[m]))
    print(f"{builder} a={scale:+.1f} qLogEI: rows per regime {cov.count}, per eighth of v {cov.eighths.tolist()}, "
          f"worst err/bound per regime {per_class}")
    cov.check(min_count=5)


def test_near_tie_at_the_threshold_keeps_the_17th_sample_in_the_table(cuda_device):
    """A 17th-largest sample one ulp below the 16th belongs to the tail.  The tables used to test it as
    zeta - w < zeta_(16) - w, rounded, and dropped it from every entry with large w: up to 1/(S - 16) of the tail."""
    for builder in ("cta", "grid", "wide"):
        gp, x = _model(builder, cuda_device)
        mu, var = _moments(gp, x)
        z = ar.make_samples("near_tie16", 64, 1.0, seed=7)
        top, ok = ar.table_head(z, 1.0)
        assert ok
        mo = mu.astype(np.float64) + SHIFT
        so = np.sqrt(var.astype(np.float64))
        acq = AcqConfig(kind="qLogEI", best_f=float(np.median(mo + so * (top[0] + 60))), obj_shift=SHIFT)
        got, _ = _score(gp, acq, x, z)
        ref, bound = ar.mc_bound(acq, mu, var, z, "fused", table_on=True)
        _check(f"{builder} near tie", got, ref, bound)
        cls, _ = ar.classify(acq, mu, var, z)
        assert (cls == ar.FAST).sum() > 100


# ------------------------------------------------------------------------------------------------------------------
# bb_acq_score on synthetic moments
# ------------------------------------------------------------------------------------------------------------------
MOMENT_S = [1, 2, 31, 32, 33, 100, 511, 1023, 1024]


def _synthetic_rows(acq):
    """fp32 (mu, var): analytic u = (mo - best_f)/s over [-1e7, 40] with points on both sides of -1 and -1e6, var
    from the 1e-10 clamp to 100, and rows at mo == best_f exactly."""
    p = ar.spec32(acq)
    u = np.concatenate([-np.geomspace(1e-3, 1e7, 90), np.linspace(-3, 40, 60),
                        [-1 - 1e-6, -1.0, -1 + 1e-6, -0.999, -1.001, -1e6 * (1 + 1e-5), -1e6, -1e6 * (1 - 1e-5)]])
    rows_mu, rows_var = [], []
    for var in (1e-10, 1e-4, 1.0, 100.0):
        s = abs(p["obj_scale"]) * np.sqrt(np.float64(F32(var)))
        mo = p["best_f"] + u * s
        rows_mu.append(((mo - p["obj_shift"]) / p["obj_scale"]).astype(F32))
        rows_var.append(np.full(u.size, var, F32))
    mu0 = F32(0.5)  # mo == best_f exactly: the best_f of the spec is set to fma(a, 0.5, b), exact in fp32
    rows_mu.append(np.full(4, mu0))
    rows_var.append(np.array([1e-10, 1e-4, 1.0, 100.0], F32))
    return np.concatenate(rows_mu), np.concatenate(rows_var)


def _spec_at_exact_incumbent(kind, scale, **kw):
    bf = float(F32(scale) * F32(0.5) + F32(SHIFT))
    assert float(F32(bf)) == bf
    return AcqConfig(kind=kind, best_f=bf, beta=0.3, obj_scale=scale, obj_shift=SHIFT, **kw)


@pytest.mark.parametrize("scale", SCALES)
def test_acq_score_analytic_kinds_on_synthetic_moments(scale, cuda_device):
    for kind in ANALYTIC_KINDS:
        acq = _spec_at_exact_incumbent(kind, scale)
        mu, var = _synthetic_rows(acq)
        got = _acq_score(acq, mu, var, None, cuda_device)
        ref = ar.analytic_ref(acq, mu, var)
        assert np.isfinite(ref).all()
        r = _check(f"acq_score {kind} a={scale}", got, ref, ar.analytic_bound(ref))
        print(f"acq_score a={scale:+.1f} {kind}: worst err/bound {r:.3f}")


@pytest.mark.parametrize("kind", MC_KINDS)
@pytest.mark.parametrize("scale", SCALES)
def test_acq_score_mc_kinds_on_synthetic_moments(kind, scale, cuda_device):
    worst = {}
    for S in MOMENT_S:
        for name in ("sobol", "normal", "heavy"):
            z = ar.make_samples(name, S, 1.0, seed=S)
            acq = _spec_at_exact_incumbent(kind, scale)
            mu, var = _synthetic_rows(acq)
            got = _acq_score(acq, mu, var, z, cuda_device)
            ref, bound = ar.mc_bound(acq, mu, var, z, "moments")
            worst[S] = max(worst.get(S, 0.0), _check(f"acq_score {kind} S={S} {name}", got, ref, bound))
    print(f"acq_score {kind} a={scale:+.1f}: worst err/bound per S {worst}")


def test_qlogei_fp32_domain_edge(cuda_device):
    """qLogEI's float64 value stays finite however far a row lies below the incumbent; in fp32 1/(1+t^2) flushes
    to zero once every sample has |t| >= 2^63 (9.2e18), and the kernel returns -inf there (the documented domain
    of acq_math.cuh's mc_finalize).  Closer rows stay within the bound."""
    z = ar.make_samples("sobol", 64, 1.0)
    acq = AcqConfig(kind="qLogEI", best_f=0.0)
    gaps = np.array([1e11, 1e12, 5e12, 9e12, 1e13, 2e13, 1e14], np.float64)  # best_f - mo; t = -gap / tau
    mu = (-gaps).astype(F32)
    var = np.full(gaps.size, 1.0, F32)
    got = _acq_score(acq, mu, var, z, cuda_device)
    ref, bound = ar.mc_bound(acq, mu, var, z, "moments")
    assert np.isfinite(ref).all()
    c0, c1 = ar.coefs32(acq, mu, var)
    tmax = np.abs(c0.astype(np.float64)[:, None] + c1.astype(np.float64)[:, None] * z[None, :]).min(1)
    outside = tmax >= 2.0**63
    assert outside.any() and (~outside).any()
    assert np.all(got[outside] == -np.inf), got
    _check("qLogEI inside the fp32 domain", got[~outside], ref[~outside], bound[~outside])


# ------------------------------------------------------------------------------------------------------------------
# arg-max keys
# ------------------------------------------------------------------------------------------------------------------
def _expected_order(s: np.ndarray, keep=None):
    """Indices by (score descending, index ascending), NaN and masked rows skipped; -0.0 == +0.0."""
    ok = ~np.isnan(s)
    if keep is not None:
        ok &= keep != 0
    idx = np.nonzero(ok)[0]
    return idx[np.lexsort((idx, -(s[idx].astype(np.float64) + 0.0)))]


def _key_cases(n: int = 70_000):
    rng = np.random.default_rng(0)
    base = rng.standard_normal(n).astype(F32)
    zeros = np.where(rng.random(n) < 0.5, F32(0.0), F32(-0.0)).astype(F32)
    cases = {"random": base, "signed_zeros": zeros}
    tie = base.copy()
    top = F32(base.max() + 1)
    tie[[40_000, 300, 9_999, 65_000]] = top  # ties in different CTAs
    cases["ties_across_ctas"] = tie
    z2 = np.full(n, F32(-1.0))
    z2[[5, 70, 33_000]] = F32(-0.0)
    z2[[20_000, 500]] = F32(0.0)
    cases["zero_ties_above_negatives"] = z2
    cases["all_minus_inf"] = np.full(n, -np.inf, F32)
    nan = tie.copy()
    nan[[0, 300, 1234]] = np.nan
    cases["nan_rows"] = nan
    return cases


def test_argmax_and_topk_keys_follow_torch_semantics(cuda_device):
    n = 70_000
    keep = (np.random.default_rng(1).random(n) < 0.7).astype(np.uint8)
    keep[[300, 40_000]] = 0
    for name, s in _key_cases(n).items():
        st = torch.from_numpy(s).to(cuda_device)
        for kp in (None, keep):
            kt = None if kp is None else torch.from_numpy(kp).to(cuda_device)
            order = _expected_order(s, kp)
            for off in (0, (1 << 32) - 2 - n):
                val, idx = decode_best(torch.ops.baybe_b200.argmax(st, kt, off))
                if order.size == 0:
                    assert idx == -1, (name, off)
                    continue
                assert idx == int(order[0]) + off and val == float(s[order[0]]), (name, kp is not None, off, idx)
                if kp is None and not np.isnan(s).any():
                    assert int(order[0]) == int(torch.argmax(st).item()), name
            if order.size and np.isfinite(s[order[:5]]).all():
                k = min(5, order.size)
                vals, idx = torch.ops.baybe_b200.topk(st, kt, k)
                assert idx.cpu().tolist() == order[:k].tolist(), (name, kp is not None)
                assert np.array_equal(vals.cpu().numpy(), s[order[:k]]), name


def test_pm_with_negative_scale_scores_minus_zero_and_ties_with_plus_zero(cuda_device):
    """PM with obj_scale < 0 and obj_shift = -0.0 scores mu = +0.0 as -0.0 and mu = -0.0 as +0.0.  The two zeros
    tie: the arg-max is the lower index, as torch.argmax returns."""
    acq = AcqConfig(kind="PM", obj_scale=-0.7, obj_shift=-0.0)
    mu = np.array([1.0, 0.0, -0.0, 0.0, 2.0], F32)
    var = np.ones(5, F32)
    got = _acq_score(acq, mu, var, None, cuda_device)
    assert np.signbit(got[1]) and not np.signbit(got[2])
    st = torch.from_numpy(got.astype(F32)).to(cuda_device)
    assert decode_best(torch.ops.baybe_b200.argmax(st, None, 0))[1] == int(torch.argmax(st).item()) == 1
    vals, idx = torch.ops.baybe_b200.topk(st, None, 3)
    assert idx.cpu().tolist() == [1, 2, 3]


def test_fused_keys_with_masks_ties_and_offsets(cuda_device):
    """score_fused's key against torch.argmax of its own scores: PM ties between duplicated candidate rows in
    different tiles, keep masks, and index_offset next to the 32-bit limit."""
    w = numeric_grid_workload(N=1000, d=6, n=64, seed=11)
    cand = w.candidates.copy()
    cand[[900, 130, 777]] = cand[int(np.argmax(cand.sum(1)))]
    gp = DeviceGP(device=cuda_device, **w.gp_kwargs())
    x = gp.prepare(torch.from_numpy(cand))
    rng = np.random.default_rng(2)
    for kind, scale in (("PM", 1.0), ("PM", -0.7), ("UCB", -0.7), ("qEI", 1.0)):
        acq = AcqConfig(kind=kind, obj_scale=scale, obj_shift=SHIFT, best_f=0.3)
        z = torch.from_numpy(ar.make_samples("sobol", 64)).to(cuda_device) if acq.is_mc else None
        for keep in (None, (rng.random(1000) < 0.5).astype(np.uint8)):
            kt = None if keep is None else torch.from_numpy(keep).to(cuda_device)
            for off in (0, (1 << 32) - 2 - 1000):
                s, key = torch.ops.baybe_b200.score_fused(x, kt, z, gp.handle, _lib.ACQ_KIND[kind], acq.params(),
                                                          off, True)
                order = _expected_order(s.cpu().numpy(), keep)
                assert decode_best(key)[1] == int(order[0]) + off, (kind, scale, keep is not None, off)


# ------------------------------------------------------------------------------------------------------------------
# bb_acq_score_joint on synthetic joint moments
# ------------------------------------------------------------------------------------------------------------------
# eta of the candidate collinear with pending point 0: var = s^2 (1 + eta); at s_y = 1 these land on attempts
# 0, 1, 2, 3 of the kernel's jitter rule and on the all-fail NaN, the pivots 4x or more from zero
ETAS = [1e-3, -1e-6, -6e-6, -6e-5, -1e-3]


def _joint_case(P, s_y, seed):
    rng = np.random.default_rng(seed)
    s2 = s_y * s_y
    pcov = (s2 * (np.eye(P) + 0.2 * np.diag(rng.random(P)))).astype(F32)
    pmu = (s_y * rng.standard_normal(P)).astype(F32)
    n_gen = 24
    var = (s2 * rng.uniform(0.5, 2.0, n_gen)).astype(F32)
    cross = (s2 * 0.3 * rng.standard_normal((n_gen, P)) / np.sqrt(P)).astype(F32)
    mu = (s_y * rng.standard_normal(n_gen)).astype(F32)
    e0 = np.zeros(P, F32)
    e0[0] = F32(pcov[0, 0])
    col_var = np.array([F32(pcov[0, 0]) * (1 + eta) for eta in ETAS], F32)
    mu = np.concatenate([mu, np.full(len(ETAS), F32(0.1 * s_y))])
    var = np.concatenate([var, col_var])
    cross = np.concatenate([cross, np.tile(e0, (len(ETAS), 1))])
    return mu, var, np.ascontiguousarray(cross), pmu, pcov


@pytest.mark.parametrize("P", [1, 2, 7, 8, 31])
@pytest.mark.parametrize("s_y", [1e-3, 1.0, 1e3])
def test_acq_score_joint_within_bound_across_jitter_attempts(P, s_y, cuda_device):
    worst, attempts, oracle_gap = {}, set(), 0.0
    for S in (1, 33, 512, 1024):
        mu, var, cross, pmu, pcov = _joint_case(P, s_y, seed=P * 1000 + S)
        z = np.random.default_rng(S).standard_normal((S, P + 1)).astype(F32)
        t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda_device) for k, v in
             dict(mu=mu, var=var, cross=cross, pmu=pmu, pcov=pcov, z=z).items()}
        for kind in ("qEI", "qSR", "qUCB", "qLogEI"):
            acq = AcqConfig(kind=kind, best_f=float(0.5 * s_y), beta=0.3, obj_scale=-0.7, obj_shift=SHIFT)
            got = torch.ops.baybe_b200.acq_score_joint(t["mu"], t["var"], t["cross"], t["pmu"], t["pcov"], t["z"],
                                                      _lib.ACQ_KIND[kind], acq.params()).cpu().numpy()
            got = got.astype(np.float64)
            ref_kind = "qEI" if kind == "qLogEI" else kind
            ref, bound, att = ar.joint_ref_and_bound(AcqConfig(kind=ref_kind, best_f=acq.best_f, beta=0.3,
                                                               obj_scale=-0.7, obj_shift=SHIFT),
                                                     mu, var, cross, pmu, pcov, z)
            fail = att < 0
            assert np.all(np.isnan(got[fail])), (kind, S, "all four attempts fail: NaN expected")
            assert np.all(np.isfinite(got[~fail])), (kind, S, got[~fail])
            attempts |= set(att.tolist())
            if kind == "qLogEI":
                continue  # attempts and NaN only: the values are qLogEI's, covered with pending points elsewhere
            worst[(kind, S)] = _check(f"joint {kind} P={P} S={S} s_y={s_y:g}", got[~fail], ref[~fail],
                                      bound[~fail])
        for r in np.nonzero(att > 0)[0]:  # jitter engaged: what the oracle's float64 rule would have used instead
            A = np.block([[np.array([[var[r]]], np.float64), cross[r][None, :].astype(np.float64)],
                          [cross[r][:, None].astype(np.float64), pcov.astype(np.float64)]])
            k64, L64 = ar.joint_attempt(A, "oracle")
            kk, Lk = ar.joint_attempt(A, "kernel")
            oracle_gap = max(oracle_gap, np.inf if k64 is None else float(np.abs(L64 - Lk).max()) / s_y)
    if s_y == 1.0:
        assert attempts >= {0, 1, 2, 3, -1}, attempts
    print(f"joint P={P} s_y={s_y:g}: attempts {sorted(attempts)}, worst err/bound {max(worst.values()):.3f}, "
          f"max |L(oracle jitter) - L(kernel jitter)| / s_y at jittered rows {oracle_gap:.3g}")
