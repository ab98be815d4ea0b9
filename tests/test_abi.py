"""CPU tests of the C-ABI boundary: the shared library builds (nvcc cross-compiles without a GPU),
loads, and exports exactly the entry points include/baybe_b200.h declares; the ctypes mirrors of
the C structs have the C compiler's sizes.  No compute calls (no GPU here)."""
from __future__ import annotations

import ctypes
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
HEADER = ROOT / "include" / "baybe_b200.h"


@pytest.fixture(scope="module")
def lib():
    from baybe_b200 import _lib
    from baybe_b200.build import build

    build(verbose=False)
    return _lib.load()


def _declared_functions() -> set[str]:
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return set(re.findall(r"\b(bb_[a-z0-9_]+)\s*\(", text))


def test_every_declared_symbol_is_exported_and_bound(lib):
    from baybe_b200 import _lib

    declared = _declared_functions()
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", str(_lib.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    exported = set(re.findall(r" T (bb_[a-z0-9_]+)", out))
    assert declared <= exported, declared - exported
    assert lib.bb_abi_version() == _lib.ABI_VERSION


def test_every_scoring_kernel_instantiation_has_a_shape_case(lib):
    """Each k_fused / k_kmat_tma instantiation in the library is reached by one case of test_gpu_fused_shapes.CASES,
    which checks it against the oracle on the GPU: a new instantiation without a case fails here."""
    from baybe_b200 import _lib
    from tests.test_gpu_fused_shapes import CASES, kernel_ids

    out = subprocess.run(["nm", "-C", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    built = kernel_ids(out.splitlines())
    fused = [c.fused for c in CASES.values()]
    assert len(set(fused)) == len(fused), "two cases for one k_fused instantiation"
    tabled = set(fused) | {c.kmat for c in CASES.values() if c.kmat}
    assert built == tabled, (f"no case for {sorted(built - tabled)}; "
                             f"cases for instantiations the library lacks: {sorted(tabled - built)}")


def test_struct_layouts_match_the_c_compiler(tmp_path):
    from baybe_b200 import _lib

    src = tmp_path / "sz.c"
    src.write_text(
        '#include <stdio.h>\n#include "baybe_b200.h"\nint main(void){printf("%zu %zu %zu %zu\\n",'
        "sizeof(bb_model_desc),sizeof(bb_model),sizeof(bb_acq_spec),sizeof(bb_best));return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", str(HEADER.parent), str(src), "-o", str(exe)], check=True)
    sizes = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert sizes == [ctypes.sizeof(_lib.ModelDesc), ctypes.sizeof(_lib.Model), ctypes.sizeof(_lib.AcqSpec),
                     ctypes.sizeof(_lib.Best)]


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "c89ish.c"
    src.write_text('#include "baybe_b200.h"\nint main(void){return sizeof(bb_model) == 0;}\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", str(HEADER.parent), str(src)],
                   check=True)


def test_status_codes_and_blob_size_queries_without_gpu(lib):
    assert lib.bb_model_blob_bytes(0, 3, 1) == 0
    b1 = lib.bb_model_blob_bytes(256, 20, 1)
    b2 = lib.bb_model_blob_bytes(512, 20, 1)
    assert 0 < b1 < b2
    # argument validation happens before any CUDA call
    from baybe_b200 import _lib

    rc = lib.bb_acq_score(None, None, None, 10, None, 0, None, None)
    assert rc == _lib.BB_ERR_INVALID and b"null" in lib.bb_last_error()
    with pytest.raises(ValueError):
        _lib.check(rc, "bb_acq_score")


def test_round2_entry_points_validate_their_arguments_before_any_cuda_call(lib):
    import ctypes as C

    from baybe_b200 import _lib

    # bb_nei_reduce: the caller's GEMM buffer must hold S sample columns + m root columns per row
    rc = lib.bb_nei_reduce(None, 10, 8, 4, None, None, None, None, C.c_float(1.0), C.c_float(0.0), 5, None, None)
    assert rc == _lib.BB_ERR_INVALID and b"bad shape" in lib.bb_last_error()
    assert lib.bb_nei_reduce(None, 12, 8, 4, None, None, None, None, C.c_float(1.0), C.c_float(0.0), 0, None, None) == 0
    rc = lib.bb_nei_reduce(None, 12, 8, 4, None, None, None, None, C.c_float(1.0), C.c_float(0.0), 5, None, None)
    assert rc == _lib.BB_ERR_INVALID and b"null" in lib.bb_last_error()
    # bb_score_fused_overlapped: model / acquisition spec are checked first
    rc = lib.bb_score_fused_overlapped(None, None, None, 0, 10, 20, None, 0, None, 0, None, None, None, None, 0, None,
                                       None, 0, None, None)
    assert rc == _lib.BB_ERR_INVALID and b"missing" in lib.bb_last_error()
    # bb_allreduce_best: group sanity
    g = _lib.PeerGroup()
    g.rank, g.world = 3, 2
    rc = lib.bb_allreduce_best(C.byref(g), C.c_void_p(8), 0, C.c_void_p(8), C.c_void_p(8), None)
    assert rc == _lib.BB_ERR_INVALID and b"rank 3" in lib.bb_last_error()


def _fake_model(wide: bool, n_tasks: int):
    """A bb_model filled by hand: plausible shapes, fake non-null device pointers (never dereferenced)."""
    import ctypes as C

    from baybe_b200 import _lib

    m = _lib.Model()
    m.abi_version = _lib.ABI_VERSION
    m.n = m.n_pad = 64
    m.n_chunks = 1
    m.d = m.d_pad = 2048 if wide else 20
    m.family = _lib.KERNEL_FAMILY["rbf"]
    m.task_col = -1
    m.n_tasks = n_tasks
    m.y_std = m.prior_scale = m.r_scale = 1.0
    m.wide = int(wide)
    m.d_wide = m.d if wide else 0
    for name, ctype in _lib.Model._fields_:
        if name.startswith("d_") and ctype is C.c_void_p:
            setattr(m, name, 1 << 20)
    return m


def _call_entry(lib, entry: str, m, layout: int, ldx: int) -> int:
    import ctypes as C

    from baybe_b200 import _lib

    n = 1000
    x = out = C.c_void_p(1 << 20)
    if entry == "bb_score_fused":
        a = _lib.AcqSpec(kind=_lib.ACQ_KIND["UCB"], beta=2.0, obj_scale=1.0)
        return lib.bb_score_fused(C.byref(m), C.byref(a), x, layout, n, ldx, None, None, 0, out, out, 0, None)
    if entry == "bb_posterior":
        return lib.bb_posterior(C.byref(m), x, layout, n, ldx, out, out, None, None, None, 0, None)
    if entry == "bb_kernel_matrix":
        return lib.bb_kernel_matrix(C.byref(m), x, layout, n, ldx, out, m.n, None)
    return lib.bb_debug_posterior_simt(C.byref(m), x, layout, n, ldx, out, out, None)


_ENTRIES = ["bb_score_fused", "bb_posterior", "bb_kernel_matrix", "bb_debug_posterior_simt"]
# (entry point, wide model) -> status for bit-packed rows: the scoring kernels read them from wide models only, the
# CUDA-core kernels behind bb_debug_posterior_simt and the non-wide bb_kernel_matrix never
_BITS_STATUS = {("bb_score_fused", False): "unsupported", ("bb_posterior", False): "unsupported",
                ("bb_kernel_matrix", False): "invalid", ("bb_debug_posterior_simt", False): "invalid",
                ("bb_debug_posterior_simt", True): "invalid"}
_BAD_CANDIDATES = (
    [(e, w, "17 tasks", "unsupported") for e in _ENTRIES for w in (False, True)]
    + [(e, w, "layout 5", "invalid") for e in _ENTRIES for w in (False, True)]
    + [(e, w, "bit-packed rows", s) for (e, w), s in _BITS_STATUS.items()]
    + [(e, w, "ldx too small", "invalid") for e in _ENTRIES for w in (False, True)]
)


@pytest.mark.parametrize("entry, wide, case, status", _BAD_CANDIDATES,
                         ids=[f"{e}-{'wide' if w else 'resident'}-{c}" for e, w, c, _ in _BAD_CANDIDATES])
def test_entry_points_reject_bad_candidates_before_any_cuda_call(lib, entry, wide, case, status):
    import torch

    from baybe_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("CUDA present: the fake device pointers must never reach a GPU")
    m = _fake_model(wide, n_tasks=17 if case == "17 tasks" else 1)
    layout, ldx = _lib.LAYOUT["row_f32"], m.d
    if case == "layout 5":
        layout = 5
    elif case == "bit-packed rows":
        layout, ldx = _lib.LAYOUT["bits_u8"], m.d // 8
    elif case == "ldx too small":
        ldx = m.d - 1
    rc = _call_entry(lib, entry, m, layout, ldx)
    msg = lib.bb_last_error()
    assert rc == {"invalid": _lib.BB_ERR_INVALID, "unsupported": _lib.BB_ERR_UNSUPPORTED}[status], msg
    if case == "17 tasks":
        assert b"at most 16 tasks" in msg
    else:
        assert {"layout 5": b"layout 5", "bit-packed rows": b"bit-packed", "ldx too small": b"leading dimension"}[case] \
            in msg


def test_product_has_no_cpu_fallback():
    import torch

    from baybe_b200 import DeviceGP
    from baybe_b200.synthetic import mixed_small_workload

    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        DeviceGP(**mixed_small_workload().gp_kwargs())


def test_product_never_imports_the_oracle():
    for py in (ROOT / "baybe_b200").rglob("*.py"):
        text = py.read_text()
        assert not re.search(r"^\s*(import|from)\s+oracle\b", text, flags=re.M), py
