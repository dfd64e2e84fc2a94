"""CPU-side checks of the drop-in boundary: the shared library loads and exports every symbol
include/elliot_b200.h declares; the ctypes table mirrors the header; the product package never
touches oracle/."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "elliot_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(eb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from elliot_b200.build import build
    lib_path, _ = build()
    L = ctypes.CDLL(lib_path)
    names = _header_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/elliot_b200.h but not exported"


def test_ctypes_table_mirrors_header():
    from elliot_b200._lib import SIGNATURES
    assert sorted(SIGNATURES) == _header_functions()


def test_ctypes_table_types_read_from_header():
    from ctypes import c_char_p, c_float, c_int, c_int32, c_int64, c_size_t, c_uint32, c_uint64, c_void_p
    from elliot_b200._lib import SIGNATURES
    P = c_void_p
    assert SIGNATURES["eb_last_error"] == (c_char_p, [])
    assert SIGNATURES["eb_bpr_schedule_sampled"] == (c_int, [c_int32, c_int32, P, c_int64, c_uint64, c_uint64, P, c_size_t, P,
                                                              c_int, P])
    assert SIGNATURES["eb_slim_fit_f32"] == (c_int, [P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, c_float, c_float,
                                                      c_float, c_uint32, c_int, c_int, c_int, c_int32, P, P, P, P, P, P,
                                                      c_size_t, P])


def test_header_type_without_ctypes_mapping_raises():
    import pytest
    from elliot_b200._lib import EbError, parse_header
    with pytest.raises(EbError, match="eb_x.*long"):
        parse_header("int eb_x(long n, void *stream);")


def test_version_and_error_string_without_gpu():
    from elliot_b200._lib import lib
    assert lib().eb_version() >= 100
    assert isinstance(lib().eb_last_error(), bytes)


def test_product_never_imports_oracle():
    bad = []
    for dp, _, fs in os.walk(os.path.join(ROOT, "elliot_b200")):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dp, f), errors="replace").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M) or "liboracle" in txt \
                        or re.search(r'#include\s+".*oracle', txt):
                    bad.append(os.path.join(dp, f))
    assert not bad, bad


def test_compute_call_fails_loudly_without_cuda():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from elliot_b200 import ops
    U = torch.zeros((4, 16)); b = torch.zeros(4); t = torch.zeros(4, dtype=torch.int32)
    with pytest.raises(RuntimeError):
        ops.bpr_step_f32(U, U, b, 10, t, t, t, 0.05, 0, 0, 0, 0)


def test_header_is_plain_c(tmp_path):
    """The boundary is a C ABI: include/elliot_b200.h must compile as C99 (no C++ / torch / CUDA types)."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        import pytest
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "hdr.c"
    src.write_text('#include "include/elliot_b200.h"\nint main(void) { return eb_version() < 0; }\n')
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I", root, str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
