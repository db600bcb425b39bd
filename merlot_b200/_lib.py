"""ctypes binding of include/merlot_b200.h (the C-ABI drop-in boundary).

The header is the only declaration of the ABI.  Importing this module reads it (as a C compiler sees it, comments stripped)
and turns every `typedef struct` into a ctypes.Structure under its typedef name (`merlot_gemm_t`, `merlot_attn_t`, ...);
lib() gives every `merlot_*` prototype its argtypes, restype and an errcheck, so a call with the wrong number or types of
arguments raises instead of reaching the GPU, and a negative status raises as MerlotError.  A declaration the parser does not
understand raises at import; it never guesses.

The library is the product path: if it cannot be loaded this module raises -- there is no CPU or PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libmerlot_b200.so"
HEADER_PATH = _HERE.parent / "include" / "merlot_b200.h"

MERLOT_OK = 0
MERLOT_EINVAL = -1
MERLOT_ESHAPE = -2
MERLOT_ECUDA = -3
MERLOT_ENOTIMPL = -4

GEMM_OUT_F32 = 1
GEMM_ATOMIC = 2
GEMM_GELU = 4
GEMM_MUL_DGELU = 8
GEMM_DROPOUT = 16
GEMM_GELU_GRAD_OUT = 32
GEMM_MUL_AUX = 64


class MerlotError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"merlot_b200 error {code}: {msg}")
        self.code = code


class MerlotShapeError(MerlotError, ValueError):
    """Mirrors the ValueError / assert the reference raises at graph-build time (utils/model_utils.py:29-56)."""


# The one type mapping.  Every pointer, struct pointers included, is c_void_p: callers pass device addresses as ints, None
# for NULL, or byref() of a descriptor.  The only other pointer is the `const char*` result of merlot_last_error.
_SCALARS = {"int": C.c_int, "long long": C.c_longlong, "size_t": C.c_size_t, "float": C.c_float, "double": C.c_double,
            "uint32_t": C.c_uint32, "uint64_t": C.c_uint64}
_TYPE = r"(?:const\s+)?(long long|\w+)"                                     # [const] base type
_NAMED = re.compile(_TYPE + r"(?:\s*(\*+)\s*|\s+)(\w+)")                    # [const] base [*...] name
_STRUCT = re.compile(r"typedef\s+struct\s*(?:\w+\s*)?\{([^{}]*)\}\s*(\w+)\s*;")
_PROTO = re.compile(r"(.+?)\b(merlot_\w+)\s*\((.*)\)")


def _unknown(what: str):
    return ImportError(f"{HEADER_PATH}: cannot bind {what!r}")


def _ctype(base: str, stars: str, decl: str):
    if stars:
        return C.c_void_p
    if base not in _SCALARS:
        raise _unknown(decl)
    return _SCALARS[base]


def _fields(member: str) -> list:
    """`const float *a, *b` -> [("a", c_void_p), ("b", c_void_p)]: one base type, one or more declarators."""
    first, *more = (d.strip() for d in member.split(","))
    m = _NAMED.fullmatch(first)
    if not m:
        raise _unknown(member)
    base = m[1]
    out = [(m[3], _ctype(base, m[2], member))]
    for d in more:
        m = re.fullmatch(r"(\**)\s*(\w+)", d)
        if not m:
            raise _unknown(member)
        out.append((m[2], _ctype(base, m[1], member)))
    return out


def _restype(ret: str, decl: str):
    m = re.fullmatch(_TYPE + r"\s*(\**)", ret.strip())
    if not m:
        raise _unknown(decl)
    if m[1] == "void" and not m[2]:
        return None
    if m[1] == "char" and m[2] == "*":
        return C.c_char_p
    return _ctype(m[1], m[2], decl)


def _parse(text: str):
    """{typedef name: Structure class}, {function name: (restype, argtypes)} of the header."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"#ifdef __cplusplus.*?#endif", " ", text, flags=re.S)  # the extern "C" wrapper a C compiler skips
    text = re.sub(r"^\s*#.*$", " ", text, flags=re.M)                      # include guard, #include, #define
    structs, protos = {}, {}

    def struct(m):
        fields = [f for member in m[1].split(";") if member.strip() for f in _fields(" ".join(member.split()))]
        # __slots__: assigning a misspelt field raises instead of setting a Python attribute the library never sees
        structs[m[2]] = type(m[2], (C.Structure,), {"_fields_": fields, "__slots__": ()})
        return " "

    for decl in _STRUCT.sub(struct, text).split(";"):
        decl = " ".join(decl.split())
        if not decl:
            continue
        m = _PROTO.fullmatch(decl)
        if not m:
            raise _unknown(decl)
        params = m[3].strip()
        argtypes = [] if params == "void" else [t for p in params.split(",") for _, t in _fields(p)]
        protos[m[2]] = (_restype(m[1], decl), argtypes)
    return structs, protos


_STRUCTS, _PROTOTYPES = _parse(HEADER_PATH.read_text())
globals().update(_STRUCTS)


def _errcheck(name: str, nargs: int, status: bool):
    # ctypes rejects too few arguments itself but passes surplus ones on (the call has then run with the declared ones)
    def errcheck(result, func, args):
        if len(args) != nargs:
            raise TypeError(f"{name}() takes {nargs} arguments ({len(args)} given)")
        if status and result < 0:  # header: MERLOT_OK (0) or a negative MERLOT_E* code
            check(result)
        return result
    return errcheck


_lib = None


def lib() -> C.CDLL:
    """Load libmerlot_b200.so (built in-tree by merlot_b200.build) and bind every prototype of the header.  Raises if the
    library is missing or lacks a declared symbol -- no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} not found: run `python -m merlot_b200.build` (or __graft_entry__.build()). "
            "merlot_b200 has no CPU/PyTorch fallback path.")
    l = C.CDLL(str(LIB_PATH), mode=os.RTLD_GLOBAL if hasattr(os, "RTLD_GLOBAL") else 0)
    for name, (restype, argtypes) in _PROTOTYPES.items():
        try:
            f = getattr(l, name)
        except AttributeError:
            raise ImportError(f"{LIB_PATH} does not export {name}, declared in {HEADER_PATH}") from None
        f.restype, f.argtypes = restype, argtypes
        f.errcheck = _errcheck(name, len(argtypes), restype is C.c_int)
    _lib = l
    return l


def check(rc: int) -> None:
    if rc == MERLOT_OK:
        return
    msg = lib().merlot_last_error().decode("utf-8", "replace")
    if rc == MERLOT_ESHAPE:
        raise MerlotShapeError(rc, msg)
    if rc == MERLOT_ENOTIMPL:
        raise NotImplementedError(msg)
    raise MerlotError(rc, msg)
