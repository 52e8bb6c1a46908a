"""The ctypes signatures of madrl_b200/_lib.py (SIGNATURES) against the prototypes of include/madrl_b200.h, without
a library: a wrong scalar type (an int passed where the callee reads a size_t or a double), a missing parameter or a
missing entry would otherwise only show on the device, as a truncated size or a garbage argument."""
import ctypes as C
import os
import re

from conftest import ROOT
from madrl_b200 import _lib
from test_cabi import declared_functions

SCALARS = {"int": C.c_int, "int32_t": C.c_int, "size_t": C.c_size_t, "uint64_t": C.c_uint64,
           "uint32_t": C.c_uint32, "double": C.c_double}
STRUCTS = {"madrl_ww_config": _lib.WWConfig, "madrl_ww_layout": _lib.WWLayout,
           "madrl_pursuit_config": _lib.PEConfig, "madrl_pursuit_layout": _lib.PELayout,
           "madrl_hostage_config": _lib.HWConfig, "madrl_hostage_layout": _lib.HWLayout}
RESTYPES = {("int", 0): C.c_int, ("void", 0): None, ("void", 1): C.c_void_p, ("char", 1): C.c_char_p,
            ("uint64_t", 0): C.c_uint64}


def _type(tokens):
    """(base type, pointer depth) of a declaration's type tokens, qualifiers dropped."""
    words = [t for t in tokens if t not in ("*", "const")]
    return " ".join(words), tokens.count("*")


def prototypes():
    """{name: ((base, depth) of the return type, [(base, depth) of every parameter])} of the header."""
    with open(os.path.join(ROOT, "include", "madrl_b200.h")) as f:
        src = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    out = {}
    for ret, name, args in re.findall(r"([\w\s*]+?)\b(madrl_\w+)\s*\(([^()]*)\)\s*;", src):
        params = []
        if args.strip() != "void":
            for a in args.split(","):
                tokens = re.findall(r"\w+|\*", a)
                params.append(_type(tokens[:-1]))           # the last token is the parameter's name
        out[name] = (_type(re.findall(r"\w+|\*", ret)), params)
    return out


def _expected_pointer(ct, base, depth):
    """A config / layout struct pointer must be POINTER of its Structure; any other pointer a c_void_p, a
    c_char_p for char data, or a POINTER of what it points at."""
    if base in STRUCTS and depth == 1:
        return ct is C.POINTER(STRUCTS[base])
    if ct is C.c_void_p or (ct is C.c_char_p and base in ("char", "unsigned char")):
        return True
    pointee = SCALARS.get(base) if depth == 1 else C.c_void_p
    return pointee is not None and ct is C.POINTER(pointee)


def test_prototype_parser_finds_every_declared_function():
    assert sorted(prototypes()) == declared_functions()


def test_table_has_one_entry_per_header_function():
    header, table = set(prototypes()), set(_lib.SIGNATURES)
    assert not header - table, "not in _lib.SIGNATURES: %s" % sorted(header - table)
    assert not table - header, "not in include/madrl_b200.h: %s" % sorted(table - header)


def test_table_entries_match_the_prototypes():
    bad = []
    for name, (ret, params) in prototypes().items():
        if name not in _lib.SIGNATURES:
            continue                                            # reported by the test above
        res, args = _lib.SIGNATURES[name]
        if ret not in RESTYPES or RESTYPES[ret] is not res:
            bad.append("%s: returns %s, declared %s" % (name, ret, res))
        if len(args) != len(params):
            bad.append("%s: %d parameters, declared %d" % (name, len(params), len(args)))
            continue
        for k, ((base, depth), ct) in enumerate(zip(params, args)):
            ok = _expected_pointer(ct, base, depth) if depth else SCALARS.get(base) is ct
            if not ok:
                bad.append("%s: parameter %d is %s%s, declared %s" % (name, k, base, "*" * depth, ct))
    assert not bad, "\n".join(bad)
