"""The C-ABI library loads on a CPU-only box and exports every symbol include/b3d.h declares."""
import ctypes
import os
import re

from conftest import PKG, ROOT


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "b3d.h")).read()
    return sorted(set(re.findall(r"B3D_API[^;]*?\b(b3d_\w+)\s*\(", text)))


def test_header_declares_symbols():
    syms = declared_symbols()
    assert "b3d_pc_project" in syms and "b3d_last_error" in syms
    assert len(syms) >= 10


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(os.path.join(PKG, "b3d", "libb3d.so"))
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"declared in b3d.h but not exported: {missing}"


def declared_parameter_counts():
    """{function: number of parameters} of every prototype in include/b3d.h."""
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b3d.h")).read(), flags=re.S)
    return {name: 0 if params.strip() in ("", "void") else params.count(",") + 1
            for name, params in re.findall(r"B3D_API[^;(]*?\b(b3d_\w+)\s*\(([^)]*)\)\s*;", text)}


def test_argtypes_match_the_header():
    """ctypes passes surplus trailing arguments without an error, so a binding whose argtypes disagree with the prototype
    would shift the arguments of its call sites instead of failing."""
    import b3d
    counts = declared_parameter_counts()
    typed = {n: len(getattr(b3d.lib, n).argtypes) for n in counts if getattr(b3d.lib, n).argtypes is not None}
    assert "b3d_conv2d_tf32" in typed and "b3d_pc_project" in typed
    bad = {n: (k, counts[n]) for n, k in typed.items() if k != counts[n]}
    assert not bad, f"(argtypes, parameters in b3d.h) differ: {bad}"


def test_error_reporting_without_gpu():
    import b3d
    # argument validation happens before any CUDA call
    rc = b3d.lib.b3d_pc_project(None, None, 1, 1, 1, 1.875, 2.0, None, None, None, None, None, None, None)
    assert rc == -1
    assert b"bad sizes" in b3d.lib.b3d_last_error()
    assert b3d.lib.b3d_version() >= 100


def test_cpu_tensors_are_rejected_loudly():
    import pytest
    import torch
    import b3d
    from utils.effective_loss_function import EffectiveLossFunction, PointCloudRender
    assert PointCloudRender is EffectiveLossFunction
    m = EffectiveLossFunction(voxel_size=32)
    with pytest.raises(b3d.B3DError, match="no CPU fallback"):
        m(torch.zeros(1, 4, 3), torch.ones(1, 4))
