"""Every prototype of include/hawq_b200.h against its ctypes binding in hawq_b200/_lib.py.  ctypes passes whatever argtypes say: an
argument dropped, added, narrowed or of the other signedness on either side would reach the library as a wrong value without any
error.  Needs neither the library nor a GPU."""
import ctypes as C
import os
import re

from hawq_b200 import _lib

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "hawq_b200.h")

# the ctypes type of each scalar C type the header uses: same width and signedness
SCALAR_CTYPES = {"int": C.c_int32, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "float": C.c_float,
                 "double": C.c_double}


def bound_alike(decl, ctype):
    """A parameter or return type of the header (`int32_t N`, `const float* mean3`, `int64_t`) against its ctypes binding: a pointer
    is bound as a pointer, a scalar as the ctypes type of the same width and signedness."""
    if "*" in decl:
        return ctype in (C.c_void_p, C.c_char_p) or issubclass(ctype, C._Pointer)
    return ctype is SCALAR_CTYPES[decl.replace("const ", "").split()[0]]


def test_every_prototype_matches_its_binding():
    header = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    protos = re.findall(r"((?:const\s+)?\w+\s*\**)\s*\b(hawq_\w+)\s*\(([^)]*)\)\s*;", header)
    assert {name for _, name, _ in protos} == set(_lib.SIGNATURES)
    for ret, name, args in protos:
        restype, argtypes = _lib.SIGNATURES[name]
        params = [a.strip() for a in args.split(",") if a.strip() not in ("", "void")]
        assert len(params) == len(argtypes), "%s: %d arguments in the header, %d bound" % (name, len(params), len(argtypes))
        assert bound_alike(ret, restype), "%s returns %s, bound as %s" % (name, ret.strip(), restype)
        for param, ctype in zip(params, argtypes):
            assert bound_alike(param, ctype), "%s: %s bound as %s" % (name, param, ctype)
