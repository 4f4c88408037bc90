"""CPU: the C-ABI library loads and exports every symbol include/fpose.h declares (no compute calls)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "fpose.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fp_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from foundationpose_b200 import _lib

    names = _declared()
    assert len(names) >= 20
    lib = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, f"declared in fpose.h but not exported: {missing}"


def test_error_string_and_counters_without_gpu():
    from foundationpose_b200 import _lib

    assert _lib.launch_count() >= 0
    assert isinstance(_lib.lib.fp_last_error(), (bytes, type(None)))


def test_product_path_has_no_cpu_fallback():
    """The engine refuses to run without a CUDA device instead of silently falling back."""
    import pytest
    import torch

    from foundationpose_b200 import _lib
    from foundationpose_b200.engine import Engine

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.FposeError):
        Engine()


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "foundationpose_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f"{f} imports the oracle"


# Entry points that need no try/catch of their own: accessors that only read or set a field, and wrappers that only call
# wrapped entry points.
_UNGUARDED_ACCESSORS = {"fp_last_error", "fp_launch_count", "fp_prof_enable", "fp_graph_captures", "fp_vis_workspace_bytes",
                        "fp_group_size", "fp_group_ctx"}
_UNGUARDED_WRAPPERS = {"fp_set_mesh", "fp_track", "fp_track_objects", "fp_track_cameras"}


def test_every_entry_point_catches_exceptions():
    """An exception (std::bad_alloc from a host-side vector, say) must not cross the C boundary and terminate the caller:
    every exported definition under csrc/ opens with FP_API_BEGIN, apart from the accessors and wrappers above."""
    csrc = os.path.join(ROOT, "foundationpose_b200", "csrc")
    # a definition at column 0 whose name starts with fp_ (internal helpers are static or inside namespace fp, indented
    # code is a call): its signature, then the first statement of its body
    definition = re.compile(r"^(?!static\b)[A-Za-z_][\w \*]*?\b(fp_[a-z0-9_]+)\(([^;{}]*?)\)\s*\{\s*(\S+)", re.M)
    opening = {}
    for f in sorted(os.listdir(csrc)):
        if f.endswith(".cu"):
            for m in definition.finditer(open(os.path.join(csrc, f)).read()):
                assert m.group(1) not in opening, f"{m.group(1)} defined twice"
                opening[m.group(1)] = (f, m.group(3))
    # the scan sees every function fpose.h declares, so none can escape it
    assert sorted(opening) == _declared()
    unguarded = [f"{name} ({f})" for name, (f, first) in sorted(opening.items())
                 if first != "FP_API_BEGIN" and name not in _UNGUARDED_ACCESSORS | _UNGUARDED_WRAPPERS]
    assert not unguarded, f"entry points whose body does not open with FP_API_BEGIN: {unguarded}"
