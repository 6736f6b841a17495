"""Every prototype in include/gut_b200.h, grt_b200.h and nht_b200.h has an entry in b200_native.SIGNATURES whose ctypes types match it
type for type, and load() binds them (no GPU needed): a wrong integer width would otherwise truncate silently on the way to the GPU."""
import ctypes as C

import pytest

from helpers import prototypes

HEADERS = ("gut_b200.h", "grt_b200.h", "nht_b200.h")


def _pointees():
    import b200_native as nat

    return {"gutb200_camera": nat.Camera, "gutb200_config": nat.Config, "grtb200_config": nat.GrtConfig, "nhtb200_config": nat.NhtConfig,
            "float": C.c_float, "int64_t": C.c_int64, "char": C.c_char}


SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float, "size_t": C.c_size_t}


def _matches(ctype, c_type: str) -> bool:
    """Does the ctypes type `ctype` pass the C type `c_type` ("const float*", "int64_t", ...) unchanged?"""
    base = c_type.replace("const", " ").replace("*", " ").split()[0]
    depth = c_type.count("*")
    if depth == 0:
        return ctype is SCALARS[base]
    if ctype is C.c_void_p or (ctype is C.c_char_p and base == "char" and depth == 1):
        return True
    if not (isinstance(ctype, type) and issubclass(ctype, C._Pointer)):
        return False
    if depth > 1:  # a pointer to pointers: the pointee is itself any pointer
        return ctype._type_ is C.c_void_p or issubclass(ctype._type_, C._Pointer)
    return ctype._type_ is _pointees().get(base)


@pytest.mark.parametrize("header", HEADERS)
def test_every_prototype_is_bound_type_for_type(header):
    import b200_native as nat

    protos = prototypes(header)
    assert len(protos) >= 5
    for name, (ret, params) in protos.items():
        assert name in nat.SIGNATURES, f"{name} ({header}) has no entry in b200_native.SIGNATURES"
        restype, argtypes = nat.SIGNATURES[name]
        assert len(argtypes) == len(params), f"{name}: {len(argtypes)} argtypes for {len(params)} parameters"
        for i, (ct, p) in enumerate(zip(argtypes, params)):
            assert _matches(ct, p), f"{name} argument {i}: {ct.__name__} does not pass `{p}`"
        if ret != "void":
            assert restype is not None and _matches(restype, ret), f"{name} returns `{ret}`, bound as {restype}"


def test_the_table_has_nothing_the_headers_do_not_declare():
    import b200_native as nat

    declared = set().union(*(prototypes(h) for h in HEADERS))
    assert set(nat.SIGNATURES) == declared
    assert set(nat.EXPORTS) | set(nat.GRT_EXPORTS) | set(nat.NHT_EXPORTS) == declared


def test_load_applies_the_table():
    import b200_native as nat

    lib = nat.load()
    for name, (restype, argtypes) in nat.SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == list(argtypes), name


def test_a_wrong_integer_width_is_caught():
    assert _matches(C.c_int64, "int64_t") and not _matches(C.c_int32, "int64_t")
    assert not _matches(C.c_int64, "int32_t") and not _matches(C.c_size_t, "int64_t") and not _matches(C.c_float, "int32_t")
    assert _matches(C.c_void_p, "const float*") and _matches(C.POINTER(C.c_float), "float*") and not _matches(C.c_int64, "float*")
    assert not _matches(C.POINTER(C.c_int32), "int64_t*") and _matches(C.POINTER(C.c_void_p), "float* const*")
