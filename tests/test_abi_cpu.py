"""The ctypes binding against the C ABI, no GPU needed: _native._declare declares exactly the functions of
include/dgcn.h, each with the header's return type and one fitting argtype per parameter, and every
`typedef struct dgcn_X` has a ctypes mirror with the header's field names in order.  A wrong or shifted argtype
would make ctypes pass a wrong value; this catches it before anything runs on a device."""
import ctypes
import os
import re
import types

import pytest

from deep_gcns_torch_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    """include/dgcn.h with its comments stripped."""
    with open(os.path.join(ROOT, "include", "dgcn.h")) as fh:
        return re.sub(r"/\*.*?\*/", "", fh.read(), flags=re.S)


def functions():
    """{name: (return type, [parameter declarations])} of every function the header declares."""
    found = re.findall(r"^(int|size_t|const char\*)\s+(dgcn_\w+)\(([^)]*)\);", header(), flags=re.M)
    out = {}
    for ret, name, params in found:
        params = " ".join(params.split())
        out[name] = (ret, [] if params == "void" else [p.strip() for p in params.split(",")])
    return out


def structs():
    """{name: [field names in order]} of every `typedef struct dgcn_X { ... } dgcn_X;`."""
    out = {}
    for name, body in re.findall(r"typedef struct (dgcn_\w+) \{([^}]*)\}", header()):
        fields = []
        for decl in (d.strip() for d in body.split(";") if d.strip()):
            fp = re.search(r"\(\*(\w+)\)", decl)          # function pointer member
            if fp:
                fields.append(fp.group(1))
                continue
            first, *more = decl.split(",")
            fields += [first.split()[-1].lstrip("*")] + [m.strip().lstrip("*") for m in more]
        out[name] = fields
    return out


def mirror(struct):
    """The ctypes mirror of dgcn_X in _native: dgcn_basic_conv -> BasicConvC."""
    return getattr(_native, "".join(w.capitalize() for w in struct[len("dgcn_"):].split("_")) + "C")


class _FakeLib:
    """Records what _native._declare sets, so the declarations can be read without the built library."""

    def __init__(self):
        object.__setattr__(self, "fns", {})

    def __getattr__(self, name):
        return self.fns.setdefault(name, types.SimpleNamespace())


def declared():
    lib = _FakeLib()
    _native._declare(lib)
    return lib.fns


_SCALAR = {"int": ctypes.c_int, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t,
           "float": ctypes.c_float, "double": ctypes.c_double}
_RESTYPE = {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "const char*": ctypes.c_char_p}


def _fits(param, argtype):
    m = re.fullmatch(r"(const )?(\w+)\s*(\*?)\s*\w+", param)
    assert m, "unparsed parameter %r" % param
    const, base, ptr = bool(m.group(1)), m.group(2), bool(m.group(3))
    if not ptr:
        return argtype is (ctypes.c_void_p if base == "dgcn_stream_t" else _SCALAR[base])
    if base.startswith("dgcn_"):
        return const and argtype is ctypes.POINTER(mirror(base))
    if base == "char":
        return const and argtype is ctypes.c_char_p
    return argtype is ctypes.c_void_p or (base in _SCALAR and argtype is ctypes.POINTER(_SCALAR[base]))


def test_binding_declares_exactly_the_header_functions():
    fns = functions()
    assert len(fns) >= 20
    assert set(declared()) == set(fns)


@pytest.mark.parametrize("name", sorted(functions()))
def test_signature_matches_header(name):
    ret, params = functions()[name]
    fn = declared()[name]
    assert fn.restype is _RESTYPE[ret], (name, fn.restype)
    argtypes = getattr(fn, "argtypes", None)
    assert argtypes is not None, "%s: no argtypes declared" % name
    assert len(argtypes) == len(params), (name, len(argtypes), len(params))
    for i, (p, t) in enumerate(zip(params, argtypes)):
        assert _fits(p, t), "%s argument %d: %r declared as %r" % (name, i, p, t)


@pytest.mark.parametrize("name", sorted(structs()))
def test_struct_fields_match_header(name):
    assert [f[0] for f in mirror(name)._fields_] == structs()[name]
