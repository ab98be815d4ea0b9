"""qNEHVI on the device: bb_hvi_decompose against box_decomposition (the same boxes as sets, exactly; the hypervolume
to 1e-12 relative) over M = 2, 3, 4, random, degenerate and simplex fronts, S = 1024 and the overflow; the scorer row
by row against the float64 definition fed with the device's own decompositions; the 1M-row recommendation; and real
Campaign runs."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from baybe_b200 import DeviceGP, nehvi
from baybe_b200 import multiobjective as mo
from baybe_b200.engine import AcqConfig, unpack_best
from baybe_b200.synthetic import numeric_grid_workload, smooth_target
from tests.test_gpu_mo import _same_winner
from tests.test_mo import _hvi_score_f64

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _decompose(pts: np.ndarray, ref: np.ndarray, stride: int = 1024, counts=None):
    x = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32)).to(DEV)
    cnt = None if counts is None else torch.from_numpy(np.asarray(counts, dtype=np.int32)).to(DEV)
    lo, up, n, hv = torch.ops.baybe_b200.hvi_decompose(x, cnt, [float(r) for r in ref], stride)
    return lo.cpu().numpy(), up.cpu().numpy(), n.cpu().numpy(), hv.cpu().numpy()


def _boxes(lo, up):
    return sorted(map(tuple, np.concatenate([lo, up], 1).astype(np.float64).tolist()))


def _check_same(pts, ref, counts=None):
    lo, up, n, hv = _decompose(pts, ref, counts=counts)
    for s in range(len(pts)):
        k = len(pts[s]) if counts is None else counts[s]
        p64 = pts[s, :k].astype(np.float32).astype(np.float64)
        hlo, hup, hhv = mo.box_decomposition(p64, ref)
        assert n[s] == len(hlo), (s, n[s], len(hlo))
        host = _boxes(hlo.astype(np.float32), hup.astype(np.float32))  # the layout bb_hvi_score reads: float32
        assert _boxes(lo[s, :n[s]], up[s, :n[s]]) == host, s
        assert abs(hv[s] - hhv) <= 1e-12 * max(abs(hhv), 1e-300), (s, hv[s], hhv)
    return n


def test_shared_memory_just_below_and_above_48_kb_at_four_targets():
    """The first M = 4 launches of the module: n = 22 needs 23^3 * 4 = 48668 B of dynamic shared memory, which with
    the kernel's static part is over 48 KB, then n = 23 and 31.  Each decomposes, and two calls on the same points
    write the same boxes in the same order."""
    rng = np.random.default_rng(22)
    for n in (22, 23, 31):
        pts = rng.dirichlet(np.ones(4), size=(6, n))
        _check_same(pts, np.zeros(4))
        (lo1, up1, n1, hv1), (lo2, up2, n2, hv2) = _decompose(pts, np.zeros(4)), _decompose(pts, np.zeros(4))
        assert np.array_equal(n1, n2) and np.array_equal(hv1, hv2)
        for s in range(len(pts)):  # the slots past n_cells are never written
            assert np.array_equal(lo1[s, :n1[s]], lo2[s, :n1[s]]) and np.array_equal(up1[s, :n1[s]], up2[s, :n1[s]])


@pytest.mark.parametrize("M", [2, 3, 4])
def test_decomposition_equals_the_host_decomposition(M):
    rng = np.random.default_rng(M)
    S = 96
    n = 31 if M < 4 else 16
    pts = rng.normal(size=(S, n, M))
    counts = rng.integers(0, n + 1, size=S)
    counts[:3] = [0, 1, n]
    pts[1::4, 1] = pts[1::4, 0]  # duplicates
    pts[2::4, :4] = np.round(pts[2::4, :4])  # ties on every output
    ref = np.full(M, -0.3)
    pts[3::4, 0, 0] = ref[0]  # on the reference point in one output: dropped
    _check_same(pts, ref, counts)
    # all points dominated by one
    dom = -np.abs(rng.normal(size=(8, 12, M)))
    dom[:, 0] = 1.0
    n_dom = _check_same(dom, np.full(M, -5.0))
    assert (n_dom == M).all() if M == 2 else (n_dom >= 1).all()


@pytest.mark.parametrize("M", [2, 3, 4])
def test_simplex_fronts_give_the_largest_grid(M):
    """Points on a simplex are mutually non-dominated: 31 of them give (32)^(M-1) grid columns."""
    rng = np.random.default_rng(10 + M)
    S = 16 if M == 4 else 64  # 32^3 columns per sample at M = 4: the host side of the check is the slow one
    pts = rng.dirichlet(np.ones(M), size=(S, 31))
    _check_same(pts, np.zeros(M))


def test_1024_samples_in_one_call():
    rng = np.random.default_rng(3)
    pts = rng.normal(size=(1024, 20, 3))
    n = _check_same(pts, np.full(3, -1.0))
    assert n.min() < n.max()


def test_a_decomposition_above_the_cell_stride_is_reported_not_truncated(monkeypatch):
    """31 normal points at M = 4 decompose into about a hundred boxes (no random 31-point front tried reached the 1024
    of BB_HVI_MAX_CELLS), so the overflow is exercised with a smaller stride: the device reports the full count, the
    boxes it wrote are the host's, and the scorer turns the count into the NotImplementedError ``_padded`` raises."""
    from baybe_b200 import _lib

    pts = np.random.default_rng(7).normal(size=(4, 31, 4))
    hosts = [mo.box_decomposition(p.astype(np.float32).astype(np.float64), np.full(4, -2.0)) for p in pts]
    stride = min(len(h[0]) for h in hosts) // 2
    lo, up, n, _ = _decompose(pts, np.full(4, -2.0), stride=stride)
    for s, (hlo, hup, _) in enumerate(hosts):
        assert n[s] == len(hlo) > stride
        assert set(_boxes(lo[s], up[s])) <= set(_boxes(hlo.astype(np.float32), hup.astype(np.float32)))

    class Front:
        ref, device = np.full(4, -2.0), DEV

    monkeypatch.setattr(_lib, "HVI_MAX_CELLS", stride)
    with pytest.raises(NotImplementedError, match=f"{int(n.max())} cells"):
        nehvi.NehviScorer._decompose(Front(), pts)


# ---- the scorer -------------------------------------------------------------------------------------------------------
def _models(M, n, N, seed=0, noise=1e-3):
    w = numeric_grid_workload(N=N, d=8, n=n, seed=seed)
    kw = w.gp_kwargs()
    kw["noise"] = np.array([noise])
    ys = [smooth_target(w.train_x, seed=seed + 7 * m + 1) for m in range(M)]
    gps = [DeviceGP(device=DEV, **{**kw, "train_y": y}) for y in ys]
    return w, gps, np.stack(ys, 1)


def _scorer(w, gps, ys, prune=True):
    M = len(gps)
    a = np.array([1.0, -1.0, 1.0, -1.0][:M])
    b = np.linspace(0.0, 0.5, M)
    ref = mo.compute_ref_point(ys * a + b)
    return nehvi.NehviScorer(gps, AcqConfig(kind="qNEHVI"), a, b, ref, w.train_x, prune=prune)


def _recording(monkeypatch):
    seen = {}

    def rec(*args):
        seen["args"] = args
        return torch.ops.baybe_b200.hvi_score(*args)

    monkeypatch.setattr(nehvi, "_hvi_score", rec)
    return seen


def _ref_and_bound(args):
    """The kernel's definition in float64 at the device's own moments, samples and decompositions, and a bound for
    fp32 arithmetic: each candidate sample moves by at most e = (|C| + 4) eps32 (|mu| + |c . w| + sd |z|) per target,
    which moves an improvement by at most the change of the float64 value over the corners (mu +- e), plus 2e-4 +
    2e-4 |ref| for the fp32 sums."""
    ref = _hvi_score_f64(*[t.cpu() if torch.is_tensor(t) else t for t in args])[0].double()
    mu, var, cross, linv, w = args[:5]
    eps = 2.0 ** -24
    nc = 0 if cross is None else cross.shape[2]
    mag = mu.double().abs() + 6.0 * var.double().clamp_min(0).sqrt()
    if nc:
        mag = mag + torch.einsum("mnc,msc->mns", cross.double().abs(), w.double().abs()).amax(2)
        mag = mag + 2.0 * var.double().clamp_min(0).sqrt()  # |L^-1 c|^2 cancels against var
    e = ((nc + 4) * eps * mag).cpu()
    dev = torch.zeros_like(ref)
    for sgn in (-1.0, 1.0):
        a = list(args)
        a[0] = (mu.double().cpu() + sgn * e).float()
        a = [t.cpu() if torch.is_tensor(t) else t for t in a]
        dev = torch.maximum(dev, (_hvi_score_f64(*a)[0].double() - ref).abs())
    return ref, 2e-4 + 2e-4 * ref.abs() + 2.0 * dev


@pytest.mark.parametrize("M,P,n", [(2, 0, 30), (2, 4, 30), (3, 0, 40), (3, 3, 20), (4, 0, 12), (4, 2, 10)])
def test_device_matches_the_float64_definition_row_by_row(monkeypatch, M, P, n):
    w, gps, ys = _models(M, n, 3000, seed=M + P)
    sc = _scorer(w, gps, ys)
    X = w.candidates
    pend = X[np.random.default_rng(1).choice(len(X), P, replace=False)] if P else None
    z = sc.base_samples(128, P, seed=3)
    seen = _recording(monkeypatch)
    s, key, _ = sc.values(torch.from_numpy(X), pend, z)
    args = seen["args"]
    assert args[6].shape[0] == 128  # one decomposition per sample
    dev = s.double().cpu()
    ref, bound = _ref_and_bound(args)
    err = (dev - ref).abs()
    assert bool((err <= bound).all()), f"max err {float(err.max()):.3e}, worst row {int((err - bound).argmax())}"
    i_dev = unpack_best(int(key.item()))[1]
    assert i_dev == int(torch.argmax(dev))
    assert _same_winner(i_dev, int(torch.argmax(ref)), ref, bound)
    # the device decompositions are the host's, sample by sample
    rows, _, _, o, _ = sc.conditioning(pend, None, z.double().numpy())
    lo, up, cnt = (t.cpu().numpy() for t in args[6:9])
    for k in range(0, 128, 17):
        hlo, hup, _ = mo.box_decomposition(o[k].astype(np.float32).astype(np.float64), sc.ref)
        assert _boxes(lo[k, :cnt[k]], up[k, :cnt[k]]) == _boxes(hlo.astype(np.float32), hup.astype(np.float32))


@pytest.mark.parametrize("M", [2, 3])
def test_joint_value_is_the_kernel_value_plus_the_batch_points_gain(monkeypatch, M):
    """joint_value([x, o]) = (kernel value of x over the decompositions of F_s u O_s) + mean_s(hv(F_s u O_s) - hv(F_s)):
    the kernel part against the float64 definition at the recorded inputs within its fp32 bound, the gain recomputed on
    the host from the same float32 points with ``box_decomposition`` (the device hypervolumes agree to 1e-12)."""
    w, gps, ys = _models(M, 20, 500, seed=4)
    sc = _scorer(w, gps, ys)
    X = w.candidates
    seen = _recording(monkeypatch)
    v2 = sc.joint_value(X[[10, 200]], None, seed=2, n_samples=128)
    ref, bound = _ref_and_bound(seen["args"])
    z = sc.base_samples(128, 1, seed=2).double().numpy()
    rows, _, _, o, _ = sc.conditioning(None, X[[200]], z)
    nc = len(rows)
    f32 = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    gain = np.mean([mo.box_decomposition(f32(o[s]), sc.ref)[2] - mo.box_decomposition(f32(o[s, :nc - 1]), sc.ref)[2]
                    for s in range(128)])
    assert gain > 0
    assert abs(v2 - (float(ref[0]) + gain)) <= float(bound[0]) + 1e-10 * gain, (v2, float(ref[0]), gain)
    lo, up, cnt = (t.cpu().numpy() for t in seen["args"][6:9])
    for k in range(0, 128, 9):  # the kernel part scored against the decompositions of F_s u O_s
        hlo, hup, _ = mo.box_decomposition(f32(o[k]), sc.ref)
        assert _boxes(lo[k, :cnt[k]], up[k, :cnt[k]]) == _boxes(hlo.astype(np.float32), hup.astype(np.float32))


def test_one_million_candidates_two_targets(monkeypatch):
    """1M x 20D, n = 256, S = 512, two targets, pruned baseline: the device's recommended row is the float64
    definition's over all rows (same moments, conditioning, samples and decompositions, float64 on the device)."""
    w = numeric_grid_workload(N=1_000_000, d=20, n=256, seed=0)
    kw = w.gp_kwargs()
    ys = np.stack([smooth_target(w.train_x, seed=7 * m + 1) for m in range(2)], 1)
    gps = [DeviceGP(device=DEV, **{**kw, "train_y": ys[:, m]}) for m in range(2)]
    sc = _scorer(w, gps, ys)
    z = sc.base_samples(512, 0, seed=1234)
    seen = _recording(monkeypatch)
    x32 = torch.from_numpy(w.candidates).to(DEV, torch.float32)
    s, key, _ = sc.values(x32, None, z)
    i_dev = unpack_best(int(key.item()))[1]
    assert i_dev == int(torch.argmax(s))
    mu, var, cross, linv, wts, zz, lo, up, cnt = seen["args"][:9]
    nc = cross.shape[2]
    a = torch.tensor(sc.a, device=DEV)
    b = torch.tensor(sc.b, device=DEV)
    zx = torch.stack([zz[:, m * (nc + 1) + nc] for m in range(2)], 1).double()
    ref = torch.empty(len(x32), dtype=torch.float64, device=DEV)
    lo64, up64 = lo.double(), up.double()
    C = int(cnt.max())
    valid = (torch.arange(C, device=DEV)[None, :] < cnt[:, None]).double()  # [S, C]
    r2 = [((cross[m].double() @ linv[m].double().T) ** 2).sum(1) for m in range(2)]
    step = 2048
    for c0 in range(0, len(x32), step):
        sl = slice(c0, c0 + step)
        Y = []
        for m in range(2):
            sd = (var[m, sl].double() - r2[m][sl]).clamp_min(0).sqrt()
            Y.append(mu[m, sl].double()[None] + wts[m].double() @ cross[m, sl].double().T + sd[None] * zx[:, m:m + 1])
        Y = torch.stack(Y, -1) * a + b  # [S, rows, 2]
        side = (torch.minimum(Y[:, :, None, :], up64[:, None, :C]) - lo64[:, None, :C]).clamp_min(0).prod(-1)
        ref[sl] = (side * valid[:, None, :]).sum(-1).mean(0)
    i_ref = int(torch.argmax(ref))
    if i_dev != i_ref:  # only a tie within the stated bounds of the two rows is accepted
        a2 = list(seen["args"])
        rows = [i_dev, i_ref]
        a2[0], a2[1], a2[2] = mu[:, rows], var[:, rows], cross[:, rows]
        r2_, b2 = _ref_and_bound(a2)
        assert float(r2_[1] - r2_[0]) <= float(b2[0] + b2[1]), (i_dev, i_ref, float(ref[i_dev]), float(ref[i_ref]))


@pytest.mark.parametrize("n_targets", [2, 3])
def test_nehvi_campaigns_on_the_device(monkeypatch, n_targets):
    root = Path(__file__).resolve().parents[1]
    ref_dir = root / "oracle" / "_ref"
    if not (ref_dir / "baybe").is_dir():
        pytest.skip("the reference package (baybe) is not installed under oracle/_ref")
    for p in (str(root / "tests" / "shims"), str(ref_dir)):
        if p not in sys.path:
            sys.path.append(p)
    import baybe  # noqa: F401
    from baybe.acquisition.acqfs import qNoisyExpectedHypervolumeImprovement

    from baybe_b200 import baybe_plugin
    from tests.test_mo import check_subset_batch_wins
    from tests.test_nehvi import check_nehvi_flow

    camp = check_nehvi_flow(baybe_plugin, monkeypatch, n_targets, tol=1e-4)
    assert isinstance(camp.recommender._scorer, nehvi.NehviScorer)
    if n_targets == 2:
        check_subset_batch_wins(baybe_plugin, monkeypatch, np.random.default_rng(5),
                                qNoisyExpectedHypervolumeImprovement())
