"""The ctypes declarations of terrain_diffusion_b200/_lib.py against the prototypes of include/tdx.h.

The package passes plain Python ints and None to libtdx, so the declared argtypes are what make a call correct: a
missing argtype passes a pointer above 2^31 as a C int, and a width that differs from the header (c_int32 for an
int64_t) works for small values and corrupts large ones.  Every `tdx_*` prototype is parsed from the header (comments
stripped, `const` ignored) and compared with its declaration: argument count, the ctypes size and signedness of every
value argument, a pointer type for every pointer argument, and the restype."""
import ctypes as C
import re
from pathlib import Path

import pytest

from terrain_diffusion_b200 import _lib as L

HEADER = Path(__file__).resolve().parent.parent / "include" / "tdx.h"

# header value type -> (kind, size, signed) as _kind reports it for the matching ctypes type
VALUE_TYPES = {
    "int": ("int", 4, True), "int32_t": ("int", 4, True), "uint32_t": ("int", 4, False),
    "int64_t": ("int", 8, True), "uint64_t": ("int", 8, False), "float": ("float", 4), "double": ("float", 8),
}
POINTER = ("pointer",)


def _source() -> str:
    text = re.sub(r"/\*.*?\*/", " ", HEADER.read_text(), flags=re.S)
    text = re.sub(r"//[^\n]*", " ", text)
    return re.sub(r"^\s*#[^\n]*", " ", text, flags=re.M)


def _c_type(decl: str, has_name: bool):
    """(kind, ...) of one C declaration ("const float* x", "int32_t h", "void* stream", or a bare return type)."""
    decl = re.sub(r"\bconst\b", " ", decl)
    if "*" in decl or "[" in decl:
        return POINTER
    words = decl.split()
    base = " ".join(words[:-1] if has_name else words)
    if base not in VALUE_TYPES:
        raise ValueError(f"tdx.h: no ctypes equivalent listed for {base!r} (in {decl.strip()!r})")
    return VALUE_TYPES[base]


def header_prototypes() -> dict:
    """name -> (return kind or None for void, [argument kinds])."""
    protos = {}
    for ret, name, params in re.findall(r"(?<=[;{}])\s*([^;{}()]*?)\b(tdx_\w+)\s*\(([^()]*)\)\s*;", _source()):
        params = params.strip()
        args = [] if params in ("", "void") else [_c_type(p, True) for p in params.split(",")]
        protos[name] = (None if ret.strip() == "void" else _c_type(ret, False), args)
    return protos


def _kind(t):
    """(kind, ...) of a ctypes type: ("pointer",), ("int", size, signed), ("float", size) or ("other", t)."""
    if t in (C.c_void_p, C.c_char_p) or (isinstance(t, type) and issubclass(t, C._Pointer)):
        return POINTER
    if t in (C.c_float, C.c_double):
        return ("float", C.sizeof(t))
    if isinstance(t, type) and issubclass(t, C._SimpleCData) and t._type_ in "bBhHiIlLqQ":
        return ("int", C.sizeof(t), t(-1).value < 0)
    return ("other", t)


PROTOTYPES = header_prototypes()


def test_every_tdx_function_in_the_header_is_parsed():
    names = set(re.findall(r"\b(tdx_\w+)\s*\(", _source()))
    assert len(names) >= 50
    assert set(PROTOTYPES) == names, sorted(names ^ set(PROTOTYPES))


@pytest.mark.parametrize("name", sorted(PROTOTYPES))
def test_declaration_matches_header(name):
    ret, args = PROTOTYPES[name]
    fn = getattr(L.lib(), name)
    assert fn.argtypes is not None, f"{name}: no argtypes declared"
    declared = [_kind(t) for t in fn.argtypes]
    assert len(declared) == len(args), f"{name}: {len(declared)} argtypes, the header has {len(args)} arguments"
    for i, (want, got) in enumerate(zip(args, declared)):
        assert got == want, f"{name} argument {i}: header {want}, ctypes {got} ({fn.argtypes[i]})"
    got_ret = None if fn.restype is None else _kind(fn.restype)
    assert got_ret == ret, f"{name} restype: header {ret}, ctypes {got_ret} ({fn.restype})"
