"""CPU: libimb.so loads and exports every symbol include/imb.h declares, and the ctypes binding in _lib.py declares what
the header declares: each entry point's return and argument types, each descriptor struct's fields, and the constants
(no compute calls)."""
import ctypes as C
import os
import re

from imitation_b200 import _build, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the header's descriptor structs and the ctypes.Structure that mirrors each
STRUCTS = {"imb_mlp": _lib.Mlp, "imb_disc_desc": _lib.DiscDesc, "imb_adam": _lib.Adam,
           "imb_policy_desc": _lib.PolicyDesc, "imb_env_desc": _lib.EnvDesc, "imb_ppo_hparams": _lib.PpoHparams,
           "imb_pref_unc_desc": _lib.PrefUncDesc, "imb_rollout_members": _lib.RolloutMembers,
           "imb_sync_desc": _lib.SyncDesc}
SCALARS = {"int": C.c_int32, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "float": C.c_float}
TYPE = r"(?:const\s+)?\w+\s*\**"  # a C type as the header writes it: `int64_t`, `const imb_disc_desc*`, `float*`


def _header() -> str:
    """include/imb.h with its comments removed."""
    src = open(os.path.join(ROOT, "include", "imb.h")).read()
    return re.sub(r"/\*.*?\*/", " ", src, flags=re.S)


def _ctype(decl: str):
    """The ctypes type the binding uses for a C type: scalars by width; a descriptor struct as its ctypes.Structure
    and a pointer to one as POINTER to it; `const char*` as c_char_p; every other pointer (data, stream) as c_void_p."""
    t = re.sub(r"\bconst\b|\s", "", decl)
    if t.endswith("*"):
        base = t[:-1]
        if base in STRUCTS:
            return C.POINTER(STRUCTS[base])
        return C.c_char_p if base == "char" else C.c_void_p
    return STRUCTS[t] if t in STRUCTS else SCALARS[t]


def _defines(src: str) -> dict:
    return {k: int(v) for k, v in re.findall(r"^#define[ \t]+(IMB_\w+)[ \t]+(\d+)\b", src, re.M)}


def test_library_builds_and_exports_header_symbols():
    _build.build()
    lib = _lib.lib()
    header = open(os.path.join(ROOT, "include", "imb.h")).read()
    declared = set(re.findall(r"\b(imb_[a-z_0-9]+)\s*\(", header))
    declared -= {"imb_mlp", "imb_disc_desc"}
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in imb.h but not exported"
    assert set(_lib.SYMBOLS) == declared
    for name, (restype, argtypes, _) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, f"{name}: table not applied"
    assert lib.imb_version() >= 1


def test_signature_table_matches_header_prototypes():
    protos = re.findall(rf"^\s*({TYPE})\s*\b(imb_\w+)\s*\(([^)]*)\)\s*;", _header(), re.M)
    assert len(protos) > 40, "prototypes not parsed"
    assert list(_lib.SIGNATURES) == [name for _, name, _ in protos], "entry points differ from imb.h (or their order)"
    for ret, name, params in protos:
        params = [] if params.strip() == "void" else params.split(",")
        want = [_ctype(re.fullmatch(rf"\s*({TYPE})\s*\w+\s*", p).group(1)) for p in params]
        restype, argtypes, kernels = _lib.SIGNATURES[name]
        assert restype is _ctype(ret), f"{name}: restype {restype.__name__}, imb.h returns {ret}"
        assert len(argtypes) == len(want), f"{name}: {len(argtypes)} argtypes, imb.h has {len(want)} parameters"
        for i, (got, w) in enumerate(zip(argtypes, want)):
            assert got is w, f"{name} argument {i} ({params[i].strip()}): {got.__name__} here, {w.__name__} in imb.h"
        assert kernels is None or (isinstance(kernels, int) and kernels >= 0), name


def _layout(t):
    """(element type, array length or None) of a ctypes field type."""
    return (t._type_, t._length_) if issubclass(t, C.Array) else (t, None)


def test_structs_match_header_layout():
    src = _header()
    defines = _defines(src)
    structs = re.findall(r"typedef\s+struct\s+(\w+)\s*\{(.*?)\}\s*\1\s*;", src, re.S)
    assert sorted(name for name, _ in structs) == sorted(STRUCTS)
    for sname, body in structs:
        want = []
        for decl in filter(str.strip, body.split(";")):
            ctype, names = re.fullmatch(rf"\s*({TYPE})\s*(.+?)\s*", decl, re.S).groups()
            for n in names.split(","):
                field, dim = re.fullmatch(r"\s*(\w+)\s*(?:\[\s*(\w+)\s*\])?\s*", n).groups()
                length = None if dim is None else int(dim) if dim.isdigit() else defines[dim]
                want.append((field, _ctype(ctype), length))
        got = [(field, *_layout(t)) for field, t in STRUCTS[sname]._fields_]
        assert got == want, f"{sname} differs from {STRUCTS[sname].__name__}"


def test_constants_match_header():
    src = _header()
    consts = _defines(src)
    consts.update((k, int(v)) for k, v in re.findall(r"\b(IMB_ST_\w+)\s*=\s*(\d+)", src))
    assert "IMB_ST_WORDS" in consts and "IMB_PU_MAX_MEMBERS" in consts, "constants not parsed"
    for name, value in consts.items():
        got = getattr(_lib, name, getattr(_lib, name[len("IMB_"):], None))
        assert got == value, f"{name} = {value} in imb.h, {got} in _lib"


def test_struct_sizes_match_header_layout():
    assert C.sizeof(_lib.Mlp) == 40
    assert C.sizeof(_lib.DiscDesc) == 24 + 40 + 4 + 40 + 12
    assert C.sizeof(_lib.Adam) == 20
    assert C.sizeof(_lib.EnvDesc) == 32
    assert C.sizeof(_lib.PpoHparams) == 44
    assert C.sizeof(_lib.PolicyDesc) == 4 * 20
