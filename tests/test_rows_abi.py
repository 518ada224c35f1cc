"""rcvd_row_layout / rcvd_evaluate_rows without a GPU: the refusals that need no device, the ctypes mirror of the row-layout structs
against a C compilation of include/rcvd.h, and the ABI version (a pure addition leaves version-1 callers working)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_both_calls_refuse_a_null_handle():
    from robust_cvd_b200 import abi, solver
    L = solver.lib()
    out = abi.RowLayout()
    assert L.rcvd_row_layout(None, C.byref(out)) == abi.ERR_INVALID
    assert L.rcvd_last_error().decode() == "null problem"
    r = np.zeros(3); rho = np.zeros(1); cols = np.zeros(3, np.int32); jac = np.zeros(3)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))     # noqa: E731
    for fam in (abi.ROWS_PAIRS, abi.ROWS_REGULARISERS, 7, -1):
        for args in ((p(r, C.c_double), p(rho, C.c_double), None, None),
                     (None, None, p(cols, C.c_int32), p(jac, C.c_double)),
                     (None, None, p(cols, C.c_int32), None)):
            assert L.rcvd_evaluate_rows(None, C.c_int32(fam), *args) == abi.ERR_INVALID
            assert L.rcvd_last_error().decode() == "null problem"


def test_creating_a_handle_without_a_device_fails_as_before():
    """Without a GPU no handle exists to ask for rows: creation reports RCVD_ERR_NO_DEVICE."""
    from robust_cvd_b200 import abi, solver
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(RuntimeError, match=rf"^rcvd error {abi.ERR_NO_DEVICE}: "):
        solver.Problem(abi.default_config(4, 1.5))


def test_problem_rows_rejects_an_unknown_family_name_before_the_library():
    from robust_cvd_b200 import solver
    P = solver.Problem.__new__(solver.Problem)      # no device: only the argument check runs
    with pytest.raises(ValueError):
        P.rows("edges")
    with pytest.raises(ValueError):
        P.rows(4)


def test_row_layout_structs_match_the_header(tmp_path):
    from robust_cvd_b200 import abi
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stddef.h>
#include <stdio.h>
#include "rcvd.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %d %d %d %d %d\\n", sizeof(rcvd_row_family), offsetof(rcvd_row_family, blocks),
         offsetof(rcvd_row_family, residuals), offsetof(rcvd_row_family, max_cols), sizeof(struct rcvd_row_layout),
         offsetof(struct rcvd_row_layout, family), RCVD_ROWS_PAIRS, RCVD_ROWS_TRIPLETS, RCVD_ROWS_DEPTH_PAIRS, RCVD_ROWS_REGULARISERS,
         RCVD_ROW_FAMILIES);
  return 0;
}
""")
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(abi.RowFamily), abi.RowFamily.blocks.offset, abi.RowFamily.residuals.offset, abi.RowFamily.max_cols.offset,
                   C.sizeof(abi.RowLayout), abi.RowLayout.family.offset,
                   abi.ROWS_PAIRS, abi.ROWS_TRIPLETS, abi.ROWS_DEPTH_PAIRS, abi.ROWS_REGULARISERS, len(abi.ROW_FAMILIES)]
    assert C.sizeof(abi.RowLayout) == 4 * 16


def test_abi_version_is_still_1():
    from robust_cvd_b200 import solver
    L = solver.lib()
    assert L.rcvd_abi_version() == 1
    assert hasattr(L, "rcvd_row_layout") and hasattr(L, "rcvd_evaluate_rows")
