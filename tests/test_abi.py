"""The C-ABI library loads on a CPU-only box and exports every symbol include/b200reg.h declares."""
import ctypes
import os
import re

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    with open(os.path.join(REPO, "include", "b200reg.h")) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200reg_[a-z_0-9]+)\s*\(", text)))


def test_header_symbols_are_exported():
    from b200reg.build import build_native
    lib = ctypes.CDLL(build_native())
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), "include/b200reg.h declares %s but libb200reg.so does not export it" % n
    from b200reg.native import EXPORTS
    assert set(EXPORTS) <= set(names)
    # the read-only taps of the parity tests are bound as well (index build, shared radix sort, matcher, LM controller)
    assert {"b200reg_index_tap", "b200reg_sort_tap", "b200reg_match_tap", "b200reg_lm_step_tap"} <= set(EXPORTS)


def test_no_gpu_means_loud_failure_not_fallback():
    """Without a device the product must refuse to run (no CPU fallback, no oracle behind the ABI)."""
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    import b200reg
    import pytest
    with pytest.raises(b200reg.B200RegError):
        b200reg.Context(0)


def test_struct_layouts_match_header():
    from b200reg import native
    assert ctypes.sizeof(native.GicpParams) == 56
    assert native.default_params().regularization == 3  # PLANE
    assert ctypes.sizeof(native.Result) == 16 * 8 + 16 * 4 + 16 * 8 + 36 * 8 + 8 + 8 * 4
    # the binding's layouts against what the compiler laid out (b200reg_struct_size)
    lib = native.lib()
    lib.b200reg_struct_size.restype = ctypes.c_size_t
    for which, st in enumerate((native.GicpParams, native.Result, native.QuatroParams, native.QuatroInfo, native.LoopConfig,
                                native.LoopFactor, native.LmTrial, native.LmCase, native.LmStep)):
        assert lib.b200reg_struct_size(which) == ctypes.sizeof(st), st.__name__
    assert lib.b200reg_struct_size(9) == 0
    assert ctypes.sizeof(native.LmCase) == 58 * 8 + 56 + 4 * 4 and native.LmCase.params.offset == 58 * 8
    assert ctypes.sizeof(native.LmStep) == 44 * 8 + 200 + 6 * 4 and native.LmStep.record.offset == 44 * 8
    assert native.Result.pose_between.offset == 192
    p = native.default_params()
    assert (p.k_correspondences, p.max_iterations, p.lm_max_iterations) == (15, 32, 10)
    assert (p.max_corr_dist, p.transformation_eps, p.rotation_eps, p.icp_score_thr) == (52.5, 0.01, 2e-3, 1.5)


def test_product_never_touches_the_oracle():
    """oracle/ is test infrastructure: nothing under the package may import, link or dlopen it."""
    pkg = os.path.join(REPO, "fast-lio-sam-qn_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp")):
                with open(os.path.join(root, f), errors="ignore") as fh:
                    t = fh.read()
                assert "liboracle" not in t and "from oracle" not in t and "import oracle" not in t, os.path.join(root, f)
