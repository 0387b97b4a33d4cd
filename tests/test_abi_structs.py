"""CPU test of the ctypes mirrors of include/pertgnn.h: every ``typedef struct`` of the header has a ``ctypes.Structure``
of the same name in pert_gnn_kdd23_b200/_lib.py with the same fields in the same order, each of the matching ctypes
type (pointers as c_void_p, fixed arrays with their lengths, nested structs as their mirrors)."""
import ctypes
import os
import re

import pytest

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pertgnn.h")
SCALARS = {"int32_t": ctypes.c_int32, "int": ctypes.c_int, "long long": ctypes.c_longlong, "float": ctypes.c_float,
           "double": ctypes.c_double}


def _structs():
    """{name: [(field, base type, is_pointer, array length or None)]} of every typedef struct of the header."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    defines = {k: int(v) for k, v in re.findall(r"#define\s+(\w+)\s+\(?(-?\d+)\)?", src)}
    out = {}
    for name, body, alias in re.findall(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*(\w+)\s*;", src, flags=re.S):
        assert name == alias, name
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            m = re.match(r"(?:const\s+)?((?:unsigned\s+)?(?:long\s+long|\w+))\s*(.*)$", decl, flags=re.S)
            assert m, decl
            base = m.group(1)
            for d in m.group(2).split(","):
                d = d.strip()
                dm = re.fullmatch(r"(\*?)\s*(\w+)(?:\[(\w+)\])?", d)
                assert dm, d
                n = dm.group(3)
                fields.append((dm.group(2), base, bool(dm.group(1)), None if n is None else int(defines.get(n, n))))
        out[name] = fields
    return out


def test_header_has_structs():
    s = _structs()
    assert {"PertModelDesc", "PertProbe", "PertStore", "PertBatchOut", "PertResourceAsOf", "PertWhatIf",
            "PertRuntimeKeys", "PertRuntimeTable", "PertChunkMix", "PertMixOut", "PertIngestState", "PertEvictOut",
            "PertSpanTable", "PertTraceGroups"} <= set(s)
    assert ("cat_rows", "int32_t", False, 4) in s["PertModelDesc"]
    assert ("keys", "PertRuntimeKeys", False, None) in s["PertIngestState"]
    assert ("h2", "uint64_t", True, None) in s["PertRuntimeTable"]


@pytest.mark.parametrize("name", sorted(_structs()))
def test_mirror_matches_header(name):
    from pert_gnn_kdd23_b200 import _lib

    mirror = getattr(_lib, name, None)
    assert isinstance(mirror, type) and issubclass(mirror, ctypes.Structure), f"_lib.{name} is missing"
    want = _structs()[name]
    got = mirror._fields_
    assert [f for f, *_ in want] == [f for f, _ in got], name
    for (field, base, ptr, n), (_, ctype) in zip(want, got):
        if n is not None:
            assert issubclass(ctype, ctypes.Array) and ctype._length_ == n, field
            ctype = ctype._type_
        if ptr:
            assert ctype is ctypes.c_void_p, field
        elif base in SCALARS:
            assert ctype is SCALARS[base], field
        else:
            assert ctype is getattr(_lib, base), field
