"""The ctypes binding takes every signature from include/mvsf_b200.h: each declared entry point is parsed, each C type
maps to one ctypes type (an unknown one is refused), and profile_calls brackets exactly the entry points that take a
stream.  No GPU needed."""
import ctypes
import inspect
import os
import re

import pytest

from mvsformerplusplus_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from mvsformerplusplus_b200.build import build
    build()
    return _lib.lib()


def test_every_declared_entry_point_is_parsed():
    header = open(os.path.join(ROOT, "include", "mvsf_b200.h")).read()
    protos = _lib.prototypes()
    assert set(protos) == set(re.findall(r"\b(mvsf_[a-z0-9_]+)\s*\(", header))
    assert protos["mvsf_last_error"] == ("const char*", [])
    assert protos["mvsf_launch_count"] == ("long long", ["int"])
    assert protos["mvsf_ktimer_read"] == ("int", ["const char*", "double*", "long long*"])
    assert protos["mvsf_fusion_filter"] == ("int", ["int"] + ["const float*"] * 4 + ["int", "int", "const int*"] +
                                            ["int"] * 3 + ["float"] * 5 +
                                            ["unsigned char*", "float*", "void*", "size_t", "mvsf_stream_t"])
    assert protos["mvsf_fusion_extract"] == ("int", ["const unsigned char*", "const float*", "const void*", "size_t",
                                                     "const float*", "const float*", "float*", "unsigned char*",
                                                     "long long", "int", "int", "mvsf_stream_t"])


def test_every_parameter_maps_to_a_ctypes_type(lib):
    P, I, F, Z = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
    for name, (ret, params) in _lib.prototypes().items():
        fn = getattr(lib, name)
        assert fn.restype is _lib.ctype(ret) and list(fn.argtypes) == [_lib.ctype(p) for p in params], name
    assert lib.mvsf_last_error.restype is ctypes.c_char_p and list(lib.mvsf_last_error.argtypes) == []
    assert lib.mvsf_launch_count.restype is ctypes.c_longlong
    assert list(lib.mvsf_fusion_filter.argtypes) == [I, P, P, P, P, I, I, ctypes.POINTER(I), I, I, I, F, F, F, F, F, P, P,
                                                     P, Z, P]
    assert list(lib.mvsf_fusion_extract.argtypes) == [P, P, P, Z, P, P, P, P, ctypes.c_longlong, I, I, P]
    assert list(lib.mvsf_ktimer_read.argtypes) == [ctypes.c_char_p, ctypes.POINTER(ctypes.c_double),
                                                   ctypes.POINTER(ctypes.c_longlong)]


@pytest.mark.parametrize("spelling", ["double", "unsigned", "bool", "mvsf_handle_t", "const float"])
def test_unknown_type_spelling_is_rejected(spelling):
    with pytest.raises(ValueError, match="no ctypes type"):
        _lib.ctype(spelling)


def test_header_parser_spellings_and_refusals(tmp_path):
    h = tmp_path / "h.h"
    h.write_text("#include <stddef.h>\n/* int mvsf_commented(int x); */\n"
                 "int mvsf_a(const float *x, long   long n,\n  int* out, mvsf_stream_t stream);  // note\n"
                 "int mvsf_b(void);\nint mvsf_c(double d);\n")
    protos = _lib.prototypes(str(h))
    assert protos == {"mvsf_a": ("int", ["const float*", "long long", "int*", "mvsf_stream_t"]), "mvsf_b": ("int", []),
                      "mvsf_c": ("int", ["double"])}
    with pytest.raises(ValueError, match="no ctypes type"):
        _lib.ctype(protos["mvsf_c"][1][0])
    h.write_text("int mvsf_d(int (*callback)(int));\n")
    with pytest.raises(ValueError, match="cannot parse"):
        _lib.prototypes(str(h))


def test_profile_calls_wraps_exactly_the_stream_entry_points(lib):
    streamed = {n for n, (_, params) in _lib.prototypes().items() if params[-1:] == ["mvsf_stream_t"]}
    assert "mvsf_warp_corr_entropy_store" in streamed and "mvsf_fusion_filter" in streamed
    assert not streamed & {"mvsf_fpn_tc_bytes", "mvsf_fmt_workspace_bytes", "mvsf_warp_corr_plan",
                           "mvsf_attention_split_plan", "mvsf_warp_corr_set_tile_path", "mvsf_ktimer_read"}
    names = list(_lib.prototypes())
    with _lib.profile_calls():
        wrapped = {n for n in names if inspect.isfunction(getattr(lib, n))}
    assert wrapped == streamed
    assert not any(inspect.isfunction(getattr(lib, n)) for n in names)   # restored on exit


def test_call_and_size_check_the_status(lib):
    assert _lib.size("mvsf_fusion_workspace_bytes", 16, 24) == 4 * (2 + 1)
    with pytest.raises(RuntimeError, match=r"mvsf_costreg_tr_workspace_bytes failed \(status -1\): .*down_rate"):
        _lib.size("mvsf_costreg_tr_workspace_bytes", 8, 31, 16, 16)   # D not a multiple of 2
