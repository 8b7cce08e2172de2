"""The ctypes signatures come from include/cogview_b200.h (cogview_b200._lib.signatures): the parse of the real header,
a type the parser does not know, and the argument tails of the entry points that take an optional feature.  Needs
neither a GPU nor the built library."""
import ctypes
import os

import pytest

from cogview_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "cogview_b200.h")) as f:
        return f.read()


def test_one_entry_per_prototype():
    sigs = _lib.signatures(_header())
    assert len(sigs) == 64
    assert sigs["cv_version"] == (ctypes.c_int, [])
    assert sigs["cv_last_error"] == (ctypes.c_char_p, [])
    assert sigs["cv_launch_count"] == (ctypes.c_longlong, [])
    assert sigs["cv_attn_decode_workspace_bytes"] == (ctypes.c_int64, [ctypes.c_int] * 3)


def test_unknown_parameter_type_raises():
    text = "/* a comment: int cv_commented(int x); */\nint cv_fine(const float* x, int n, void* stream);\n" \
           "int cv_bogus(double scale,\n             void* stream);\n"
    with pytest.raises(_lib.CogViewB200Error, match=r"cv_bogus.*double"):
        _lib.signatures(text)
    assert list(_lib.signatures(text.replace("double", "float"))) == ["cv_fine", "cv_bogus"]


def test_feature_arguments_of_the_merged_entry_points():
    sigs = _lib.signatures(_header())
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    restype, gemm = sigs["cv_gemm_bf16"]
    assert restype is I and len(gemm) == 21
    assert gemm[-4:] == [F, ctypes.c_uint64, ctypes.c_uint32, P]          # dropout_p, seed, site, stream
    _, fwd = sigs["cv_attn_sparse_fwd"]
    assert fwd[-5:] == [F, ctypes.c_uint64, ctypes.c_uint32, P, P]        # dropout_p, seed, site, drop_mask, stream
    _, bwd = sigs["cv_attn_sparse_bwd"]
    assert bwd[-3:] == [F, P, P]                                          # dropout_p, drop_mask, stream
    _, decode = sigs["cv_attn_decode"]
    assert decode[:7] == [P, P, ctypes.c_int64, P, I, P, P]               # ..., cur_len, row_pad, out
    _, sample = sigs["cv_sample_topk"]
    assert sample[-2:] == [F, P]                                          # top_p, stream
    assert sample[6] is P                                                 # valid: the host int array


def test_no_second_entry_point_per_operation():
    sigs = _lib.signatures(_header())
    # the optional feature is an argument of the one entry point, not a twin with a suffix
    for name, twin_suffix in (("cv_gemm_bf16", "_dropout"), ("cv_attn_sparse_fwd", "_dropout"),
                              ("cv_attn_sparse_bwd", "_dropout"), ("cv_attn_decode", "_ragged"),
                              ("cv_sample_topk", "_topp")):
        assert name in sigs and name + twin_suffix not in sigs, name
    # the optimizer has only its multi-tensor forms
    for name in ("cv_adamw_step_multi", "cv_sumsq_bf16_multi"):
        assert name in sigs and name[:-len("_multi")] not in sigs, name
