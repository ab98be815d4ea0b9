"""CPU checks of the acquisition-epilogue references in tests/acq_epilogue_ref.py: the regime classifier and its
coverage check, and the qLogEI table bound against an fp32 restatement of the table path (interpolation and
the exact top 16).  The restatement stays within the bound; each planted deviation of the kernel's arithmetic
exceeds it somewhere.  The GPU side is tests/test_gpu_acq_epilogue.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from baybe_b200 import AcqConfig
from baybe_b200.engine import pack_best, unpack_best
from tests import acq_epilogue_ref as ar

F32 = np.float32
TAU = 1e-6


def _acq(sgn: float, tau: float = TAU, kind: str = "qLogEI") -> AcqConfig:
    return AcqConfig(kind=kind, best_f=0.37, obj_scale=1.0 if sgn > 0 else -0.7, obj_shift=0.25, tau_relu=tau)


def _fast_rows(acq, z, sgn, n_w: int = 160):
    """Rows inside the table's envelope: w from zeta_(9) to far above zeta_(1), sd from 1e-3 to 3."""
    top, _ = ar.table_head(z, sgn)
    ws = np.concatenate([top[ar.KMC_J] + np.geomspace(1e-4, 40.0, n_w), [top[ar.KMC_J] + 2e-6]])
    sds = np.geomspace(1e-3, 3.0, 7)
    W, SD = np.meshgrid(ws, sds)
    mu, var = ar.rows_at(acq, SD.ravel(), W.ravel())
    cls, _ = ar.classify(acq, mu, var, z)
    keep = (cls == ar.FAST) | (cls == ar.FAST_CORR)
    return mu[keep], var[keep]


def _table_scores(acq, z, mu, var, sgn_table=None, F=None, **row_kw):
    """fp32 restatement of a table row's score."""
    sgn = -1.0 if ar.spec32(acq)["obj_scale"] < 0 else 1.0
    sgn_table = sgn if sgn_table is None else sgn_table
    top, _ = ar.table_head(z, sgn_table)
    F = ar.table32(z, sgn_table) if F is None else F
    c0, c1 = ar.coefs32(acq, mu, var)
    s0, s1 = ar.row_fast32(F, top, c0, c1, **row_kw)
    s = (s0 + F32(0.1) * s1).astype(F32)
    return (F32(np.log(F32(acq.tau_relu))) + np.log(s / F32(z.size)).astype(F32)).astype(np.float64)


def _ratio(acq, z, mu, var, got):
    ref, bound = ar.mc_bound(acq, mu, var, z, "fused", table_on=True)
    return ar.worst(np.abs(got - ref), bound)


def test_classifier_places_rows_in_each_regime():
    for sgn in (1.0, -1.0):
        acq = _acq(sgn)
        z = ar.make_samples("sobol", 512, sgn)
        top, ok = ar.table_head(z, sgn)
        assert ok
        w9 = float(top[ar.KMC_J])
        #        far above     below zeta_(9)  small sd          within 30 tau of zeta_(9)
        mu, var = ar.rows_at(acq, [1.0, 1.0, 1e-4, 1.0], [w9 + 5.0, w9 - 0.5, w9 + 0.01, w9 + 5e-6])
        cls, v = ar.classify(acq, mu, var, z)
        assert list(cls) == [ar.FAST, ar.FALLBACK_T9, ar.FALLBACK_T17, ar.FAST_CORR]
        assert 0 < v[0] < 1 and v[3] > 0.999 and np.isnan(v[1])
        zt = ar.make_samples("tie16", 512, sgn)
        assert not ar.table_head(zt, sgn)[1]
        assert set(ar.classify(acq, mu, var, zt)[0]) == {ar.TABLE_OFF}
        for name in ("dup_top", "near_tie16"):
            assert ar.table_head(ar.make_samples(name, 512, sgn), sgn)[1], name


def test_coverage_fails_without_fallback_or_top_eighth():
    cov = ar.Coverage()
    cov.add(np.array([ar.FAST, ar.FAST_CORR, ar.FALLBACK_T17, ar.TABLE_OFF] * 2, dtype=object),
            np.array([k / 8 + 0.01 for k in range(8)]))
    with pytest.raises(AssertionError, match="regime classes"):
        cov.check()  # no t9 > 0 fallback row
    cov.add(np.array([ar.FALLBACK_T9], dtype=object), np.array([np.nan]))
    cov.check()
    low = ar.Coverage()
    low.add(np.array(list(ar.CLASSES), dtype=object), np.array([0.1, 0.2, 0.3, 0.5, 0.6]))
    with pytest.raises(AssertionError, match="eighths"):
        low.check()  # no row with v > 7/8


def test_reference_centre_matches_oracle():
    """The bound's corners are taken in t = c0 + c1 z; its centre is the oracle's value on the same moments."""
    acq = _acq(-1.0)
    z = ar.make_samples("normal", 100, -1.0)
    mu, var = ar.rows_at(acq, np.full(9, 0.3), np.linspace(-3, 3, 9))
    ref, _ = ar.mc_bound(acq, mu, var, z, "moments")
    c0 = (ar.spec32(acq)["obj_scale"] * mu.astype(np.float64) + ar.spec32(acq)["obj_shift"]
          - ar.spec32(acq)["best_f"]) / ar.spec32(acq)["tau_relu"]
    c1 = ar.spec32(acq)["obj_scale"] * np.sqrt(var.astype(np.float64)) / ar.spec32(acq)["tau_relu"]
    centre = ar._value_of_coefs("qLogEI", acq, c0, c1, z.astype(np.float64), z.size)
    np.testing.assert_allclose(centre, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("S", [64, 512])
@pytest.mark.parametrize("name", ["sobol", "normal", "heavy", "dup_top", "near_tie16"])
@pytest.mark.parametrize("sgn", [1.0, -1.0])
def test_table_restatement_within_bound(S, name, sgn):
    acq = _acq(sgn)
    z = ar.make_samples(name, S, sgn, seed=S)
    mu, var = _fast_rows(acq, z, sgn)
    assert mu.size > 100
    r = _ratio(acq, z, mu, var, _table_scores(acq, z, mu, var))
    print(f"S={S} {name} sgn={sgn:+.0f}: worst err/bound {r:.3f} over {mu.size} table rows")
    assert r <= 1.0


PLANTED = ["interpolation_off", "w0_from_top8", "no_tmin_correction", "tie_check_forced", "sgn_fixed_plus",
           "tail_test_on_difference"]


@pytest.mark.parametrize("fault", PLANTED)
def test_planted_table_deviation_exceeds_bound(fault):
    sgn = -1.0 if fault == "sgn_fixed_plus" else 1.0
    S = 64
    acq = _acq(sgn)
    name = {"tie_check_forced": "tie16", "tail_test_on_difference": "near_tie16"}.get(fault, "normal")
    z = ar.make_samples(name, S, sgn, seed=3)
    if fault == "tie_check_forced":  # the rows the table would take if the tie check always passed
        ok_z = ar.make_samples("normal", S, sgn, seed=3)
        mu, var = _fast_rows(acq, ok_z, sgn)
    else:
        mu, var = _fast_rows(acq, z, sgn)
    kw = {}
    if fault == "interpolation_off":
        kw = {"interpolate": False}
    elif fault == "w0_from_top8":
        kw = {"F": ar.table32(z, sgn, w0_index=ar.KMC_J - 1)}
    elif fault == "no_tmin_correction":
        kw = {"tmin_correction": False}
    elif fault == "sgn_fixed_plus":
        kw = {"sgn_table": 1.0}
    elif fault == "tail_test_on_difference":
        kw = {"F": ar.table32(z, sgn, tail_test_on_difference=True)}
    r = _ratio(acq, z, mu, var, _table_scores(acq, z, mu, var, **kw))
    print(f"{fault}: worst err/bound {r:.3g}")
    assert r > 1.0


def test_qucb_centred_on_zero_exceeds_bound():
    """qUCB's deviation term is centred on the sample mean; centring it on 0 must fail the bound."""
    acq = AcqConfig(kind="qUCB", beta=0.2, obj_scale=-0.7, obj_shift=0.25)
    z = ar.make_samples("normal", 48, 1.0, seed=1)
    mu = np.linspace(-1, 1, 11).astype(F32)
    var = np.full(11, 0.5, F32)
    ref, bound = ar.mc_bound(acq, mu, var, z, "fused")
    so = -0.7 * np.sqrt(var.astype(np.float64))
    c = np.sqrt(0.2 * np.pi / 2)
    wrong = -0.7 * mu + 0.25 + so * z.mean() + c * np.abs(so) * np.abs(z.astype(np.float64)).mean()
    assert ar.worst(np.abs(wrong - ref), bound) > 1.0


def test_log_ei_branches_agree_in_float64_near_minus_one():
    """log_ei_helper's two float64 forms agree to 1e-12 relative on [-2, -1]: moving the branch point between
    them changes no fp32 result, so that deviation is invisible to any fp32 comparison."""
    from oracle import reference_path as rp

    u = torch.linspace(-2.0, -1.0, 201, dtype=torch.float64)
    upper = torch.log(rp._phi(u) + u * rp._Phi(u))
    lower = rp._log_ei_helper(u - 0.0)  # u < -1: erfcx form
    np.testing.assert_allclose(upper[:-1].numpy(), lower[:-1].numpy(), rtol=1e-12)


def test_pack_best_orders_signed_zeros_as_equal():
    assert pack_best(-0.0, 0) > pack_best(0.0, 5)
    assert pack_best(0.0, 0) > pack_best(-0.0, 5)
    assert unpack_best(pack_best(-0.0, 3)) == (0.0, 3)
    assert pack_best(-1e-45, 0) < pack_best(-0.0, 9) and pack_best(0.0, 9) < pack_best(1e-45, 0)
    vals = [-0.0, 0.0, -0.0]
    best = max(pack_best(v, i) for i, v in enumerate(vals))
    assert unpack_best(best)[1] == int(torch.argmax(torch.tensor(vals)))
