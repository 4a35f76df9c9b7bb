"""CPU: the built shared library loads without a GPU and exports every function include/mtt_b200.h declares;
the ctypes binding (lib.py) covers exactly that set, with the header's prototypes. No compute is called."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    src = open(os.path.join(ROOT, "include", "mtt_b200.h")).read()
    return re.sub(r"/\*.*?\*/|//[^\n]*", "", src, flags=re.S)


def declared_functions():
    return sorted(set(re.findall(r"\b(mtt_[a-z0-9_]+)\s*\(", _header())))


# how a value crosses the ABI: any pointer (mtt_stream_t included), 32- or 64-bit integer, float, double or nothing
_C_CLASS = {"void": "void", "int": "i32", "int32_t": "i32", "int64_t": "i64", "size_t": "i64", "float": "f32",
            "double": "f64", "mtt_stream_t": "ptr"}


def _c_class(decl):
    """Class of a C type, with or without a parameter name ("const float* in", "int64_t ld", "void")."""
    if "*" in decl:
        return "ptr"
    return _C_CLASS[next(w for w in decl.split() if w != "const")]


def _ctypes_class(t):
    if t is None:
        return "void"
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return "ptr"
    if t._type_ in "fd":
        return "f32" if t._type_ == "f" else "f64"
    return f"i{8 * ctypes.sizeof(t)}"


def declared_prototypes():
    """name -> (return class, [argument classes]) of every mtt_* function the header declares."""
    protos = {}
    for ret, name, args in re.findall(r"^([\w \t*]+?)\b(mtt_\w+)\s*\(([^)]*)\)\s*;", _header(), flags=re.M):
        args = [a.strip() for a in args.split(",")]
        protos[name] = (_c_class(ret), [] if args == ["void"] else [_c_class(a) for a in args])
    return protos


def test_symbols_match_header_prototypes():
    """lib.SYMBOLS passes every argument with the width and kind the header declares (no built library needed)."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import lib

    protos = declared_prototypes()
    assert set(protos) == set(lib.SYMBOLS), set(protos) ^ set(lib.SYMBOLS)
    for name, (res, argtypes) in lib.SYMBOLS.items():
        want_res, want_args = protos[name]
        assert _ctypes_class(res) == want_res, f"{name}: returns {res}, header says {want_res}"
        got = [_ctypes_class(t) for t in argtypes]
        assert len(got) == len(want_args), f"{name}: {len(got)} arguments, header declares {len(want_args)}"
        for i, (g, w) in enumerate(zip(got, want_args)):
            assert g == w, f"{name}: argument {i} is {argtypes[i].__name__} ({g}), header declares {w}"


def test_library_exports_every_declared_symbol():
    import mtt_b200  # noqa: F401
    from mtt_b200 import lib

    assert os.path.exists(lib.LIB_PATH), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    cdll = ctypes.CDLL(lib.LIB_PATH)
    names = declared_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(cdll, n), f"{n} declared in include/mtt_b200.h but not exported"
    assert set(names) == set(lib.SYMBOLS), set(names) ^ set(lib.SYMBOLS)


def test_library_refuses_to_run_without_sm100():
    import mtt_b200  # noqa: F401
    from mtt_b200 import lib
    import torch

    l = lib.load()
    assert l.mtt_version() >= 100
    if not torch.cuda.is_available():
        assert l.mtt_device_check() != 0
        assert b"CUDA" in l.mtt_last_error() or b"device" in l.mtt_last_error()
