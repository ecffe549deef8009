"""The ctypes view declares every entry point of include/te_b200.h once, as the header does: the same functions, and per parameter
the ctypes kind of its C type.  A raw call through te.load_library() is then as safe as a method call, and a table line that
disagrees with the header fails here, by function and position, instead of handing a kernel a truncated address."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCALARS = {"int": C.c_int32, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "size_t": C.c_size_t,
           "double": C.c_double}
RESTYPES = {"int": C.c_int, "const char*": C.c_char_p}


def _prototypes():
    """name -> (return type, parameter declarations) of every prototype in te_b200.h, in header order."""
    src = open(os.path.join(ROOT, "include", "te_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    found = re.findall(r"\b(int|const char\s*\*)\s*(te_\w+)\s*\(([^)]*)\)\s*;", src)
    protos = {}
    for ret, name, params in found:
        params = " ".join(params.split())
        protos[name] = (" ".join(ret.split()).replace(" *", "*"), [] if params == "void" else [p.strip() for p in params.split(",")])
    # every declared name parsed, once
    assert list(protos) == re.findall(r"\b(?:int|const char\s*\*)\s*(te_\w+)\s*\(", src)
    return protos


def _kind(structs, decl):
    """The ctypes kind of one parameter: a parameter struct's pointer is POINTER(<Structure>); every other pointer or array
    (handles, void*, data) is c_void_p; scalars by SCALARS."""
    m = re.fullmatch(r"(?:const\s+)?(\w+)\s*(\**)\s*\w*\s*(\[\w*\])?", decl)
    assert m, f"unparsed parameter {decl!r}"
    base, stars, array = m.groups()
    if not stars and not array:
        assert base in SCALARS, f"no ctypes kind for {decl!r}"
        return SCALARS[base]
    if stars == "*" and not array and base in structs:
        return C.POINTER(structs[base])
    return C.c_void_p


def test_signature_table_equals_the_header(te):
    protos = _prototypes()
    table = te.capi.SIGNATURES
    only_h, only_t = sorted(set(protos) - set(table)), sorted(set(table) - set(protos))
    assert not only_h and not only_t, f"declared in te_b200.h only: {only_h}; in SIGNATURES only: {only_t}"
    assert list(table) == list(protos), "SIGNATURES is not in header order"
    structs = {"te_geometry": te.Geometry, "te_slab": te.Slab, "te_chain_params": te.ChainParams,
               "te_footprint_params": te.FootprintParams, "te_halo_peer": te.HaloPeer}
    lib = te.load_library()
    bad = []
    for name, (ret, params) in protos.items():
        fn = getattr(lib, name)
        if fn.restype is not RESTYPES[ret]:
            bad.append(f"{name}: restype {getattr(fn.restype, '__name__', fn.restype)}, the header returns {ret}")
        if fn.argtypes is None:
            bad.append(f"{name}: no argtypes")
            continue
        if len(fn.argtypes) != len(params):
            bad.append(f"{name}: {len(fn.argtypes)} argtypes, the header has {len(params)} parameters")
        for k, (got, decl) in enumerate(zip(fn.argtypes, params)):
            want = _kind(structs, decl)
            if got is not want:
                bad.append(f"{name} parameter {k} ({decl}): {got.__name__}, the header's kind is {want.__name__}")
    assert not bad, "\n".join(bad)
