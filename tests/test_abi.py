"""The C-ABI library loads and exports every symbol include/rcvd.h declares (no GPU needed)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header="rcvd.h"):
    txt = open(os.path.join(ROOT, "include", header)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(rcvd_[a-z_0-9]+)\s*\(", txt)))


def test_library_exports_declared_symbols():
    from robust_cvd_b200 import solver
    L = solver.lib()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/rcvd.h but not exported"


def test_every_exported_symbol_is_declared_in_a_header():
    """include/rcvd.h is the boundary, include/rcvd_hooks.h the test/bench hooks: nothing else is exported."""
    import subprocess
    from robust_cvd_b200 import solver
    solver.lib()
    so = os.path.join(ROOT, "robust_cvd_b200", "librcvd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True).stdout
    exported = sorted({ln.split()[-1] for ln in out.splitlines() if " T rcvd_" in ln})
    declared = set(_declared("rcvd.h")) | set(_declared("rcvd_hooks.h"))
    assert exported and not [n for n in exported if n not in declared]
    for n in _declared("rcvd_hooks.h"):
        assert n in exported, f"{n} declared in include/rcvd_hooks.h but not exported"


def test_struct_layouts_and_strides():
    from robust_cvd_b200 import abi, solver
    assert C.sizeof(abi.Config) == 19 * 4 + 4 + 12 * 8      # 19 int32 + pad + 12 doubles
    assert C.sizeof(abi.SolveSummary) == 16 + 6 * 8 + 16 + 128
    L = solver.lib()
    assert L.rcvd_abi_version() == 1
    cfg = abi.default_config(4, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=17, depth_grid_y=10)
    assert solver.frame_stride(cfg) == 7 + 170
    assert solver.depth_param_offset(cfg) == 7 and solver.spatial_param_offset(cfg) == 177
    cfg2 = abi.default_config(4, 1.5, depth_type=abi.DEPTH_GRID, depth_cubic=0, value_xform=abi.VALUE_SCALESHIFT, depth_grid_x=4, depth_grid_y=4)
    assert solver.frame_stride(cfg2) == -1      # linear grid + ScaleShift is unusable in the reference as well
    opt = abi.SolveOptions()
    L.rcvd_default_solve_options(C.byref(opt))
    assert (opt.max_iterations, opt.function_tolerance, opt.initial_radius, opt.min_relative_decrease) == (1000, 1e-6, 1e4, 1e-3)


def test_no_device_fails_loudly():
    """Without a CUDA device problem creation must fail (no CPU fallback)."""
    from robust_cvd_b200 import abi, solver
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback|no usable CUDA device"):
        solver.Problem(abi.default_config(4, 1.5))
    with pytest.raises(RuntimeError, match="no CPU fallback|no usable CUDA device"):
        solver.depth_apply(abi.default_config(1, 1.5), [1.0], [[1.0, 2.0]])


def test_filter_and_builder_fail_loudly_without_a_device():
    """No CPU fallback anywhere behind the C ABI: on a box without a usable GPU every compute entry point reports
    RCVD_ERR_NO_DEVICE with one message (skipped where a GPU is present -- the -m gpu tests cover the real calls)."""
    import numpy as np
    from robust_cvd_b200 import abi, solver
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is present")
    except ImportError:
        pass
    no_device = rf"^rcvd error {abi.ERR_NO_DEVICE}: no usable CUDA device \(.+\); this library has no CPU fallback$"
    depth = np.ones((2, 4, 4), np.float32); cams = np.zeros((2, 9), np.float32); cams[:, 6] = 1; cams[:, 7:] = 0.6
    fl = np.zeros((2, 4, 4, 2), np.float32); mk = np.full((2, 4, 4), 255, np.uint8)
    with pytest.raises(RuntimeError, match=no_device):
        solver.flow_guided_filter(depth, cams, fl, mk, fl, mk, first_out=0, num_out=2, frame_radius=1)
    with pytest.raises(RuntimeError, match=no_device):
        solver.build_constraints(np.zeros((2, 4, 4, 3), np.float32), [(0, 1)], fl[:1], mk[:1], 2, 1.0)
    grid = abi.default_config(1, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=4)
    with pytest.raises(RuntimeError, match=no_device):
        solver.depth_param_map(grid, np.ones(solver.frame_stride(grid)), 4, 4)
    plain = abi.default_config(1, 1.5)
    with pytest.raises(RuntimeError, match=no_device):
        solver.spatial_warp(plain, np.zeros(solver.frame_stride(plain)), 4, 4)
    with pytest.raises(RuntimeError, match=no_device):
        solver.static_flags(mk, 1.0, want_distance=True)
    with pytest.raises(RuntimeError, match=no_device):
        solver._check(solver.lib().rcvd_trim_device_memory(0))
    with pytest.raises(RuntimeError, match=no_device):
        solver.fp64_tensor_peaks(0)


# the A/B switches of include/rcvd_hooks.h with a valid argument list each
DEBUG_SWITCHES = [("rcvd_debug_set_order_slack", 4), ("rcvd_debug_set_overlap", 1), ("rcvd_debug_set_update_kernel", 1, 0),
                  ("rcvd_debug_set_eval_only", 0), ("rcvd_debug_set_distributed", 1), ("rcvd_debug_set_fast_path", 1)]


def test_debug_switches_report_a_null_handle():
    """Every A/B switch refuses a null handle with RCVD_ERR_INVALID and says so in rcvd_last_error(), in place of an earlier message."""
    from robust_cvd_b200 import abi, solver
    L = solver.lib()
    cfg = abi.default_config(4, 1.5)
    for name, *args in DEBUG_SWITCHES:
        with pytest.raises(RuntimeError, match="bad rank/nranks/num_sms"):      # an unrelated error first (host only)
            solver.factor_plan(cfg, [(0, 1)], num_sms=0)
        assert getattr(L, name)(None, *(C.c_int32(a) for a in args)) == abi.ERR_INVALID, name
        assert L.rcvd_last_error().decode() == "null problem", name
