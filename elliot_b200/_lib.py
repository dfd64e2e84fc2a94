"""ctypes binding of the C-ABI library.  The argument and return types of every entry point are read from its header,
include/elliot_b200.h, when this module is imported, so the header is the only declaration of the ABI.

There is NO fallback: if the shared library is missing, or no CUDA device is present when a
compute entry point is called, an exception is raised.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libelliot_b200.so")

_SCALARS = {"int": ctypes.c_int, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint32_t": ctypes.c_uint32,
            "uint64_t": ctypes.c_uint64, "float": ctypes.c_float, "double": ctypes.c_double, "size_t": ctypes.c_size_t}


class EbError(RuntimeError):
    pass


def _ctype(name, decl, ret=False):
    words = decl.replace("*", " * ").split()
    if "*" in words:
        return ctypes.c_char_p if ret and words == ["const", "char", "*"] else ctypes.c_void_p
    t = " ".join(w for w in words if w != "const")
    if t not in _SCALARS:
        raise EbError(f"{name}: no ctypes mapping for the type '{decl.strip()}'")
    return _SCALARS[t]


def parse_header(text):
    """{name: (restype, argtypes)} of every `ret eb_name(params);` in C header text.  Pointers bind as c_void_p (a
    `const char *` return as c_char_p), the fixed-width scalars as their ctypes types; any other type raises EbError."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", "", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    sigs = {}
    for stmt in re.split(r"[;{}]", text):
        m = re.fullmatch(r"\s*(.*?)\b(eb_\w+)\s*\((.*)\)\s*", stmt, flags=re.S)
        if m is None:
            continue
        ret, name, params = m.groups()
        params = [] if params.strip() == "void" else params.split(",")
        args = []
        for p in params:
            decl = re.match(r"(.*?)\w+\s*$", p, flags=re.S)
            if decl is None or not decl.group(1).strip():
                raise EbError(f"{name}: cannot read the parameter '{p.strip()}'")
            args.append(_ctype(name, decl.group(1)))
        sigs[name] = (_ctype(name, ret, ret=True), args)
    return sigs


with open(os.path.join(_HERE, "..", "include", "elliot_b200.h")) as _f:
    SIGNATURES = parse_header(_f.read())

_lib = None


def lib():
    """Load libelliot_b200.so (built by `python -m elliot_b200.build` / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EbError(f"{LIB_PATH} is missing: build it with `python -m elliot_b200.build` "
                          f"(there is no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        msg = lib().eb_last_error().decode("utf-8", "replace")
        raise EbError(f"elliot_b200 C-ABI error {rc}: {msg}")
