"""CPU-side checks of the boundary: the C-ABI library builds for sm_90a, loads, and exports
every symbol include/b200ddsp.h declares; argument errors come back as codes, not crashes.
No kernel is launched here."""
import ctypes
import re

import pytest

from ddsp_svc_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.lib()


def test_header_and_binding_agree(lib):
    hdr = open(_lib.HEADER).read()
    declared = set(re.findall(r"\b(b2d_\w+)\s*\(", hdr))
    assert declared == set(_lib.SIGNATURES)
    for name in declared:
        assert hasattr(lib, name), name


def test_binding_is_parsed_from_the_header():
    with open(_lib.HEADER) as f:
        hdr = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    parsed = _lib.prototypes(hdr, "b2d_")
    # every declaration is read: one the parser could not read would otherwise drop out of the binding silently
    assert len(parsed) == len(re.findall(r"\bb2d_\w+\s*\(", hdr)) == len(_lib.SIGNATURES)
    assert parsed["b2d_last_error"][0] is ctypes.c_char_p
    assert all(res is ctypes.c_size_t for name, (res, _) in parsed.items() if name.endswith("_workspace_bytes"))
    assert parsed["b2d_rss_loss_forward"][1][6] == (ctypes.c_void_p, "tables")          # const float* const*
    want = {"seed": ctypes.c_uint64, "ctrl_stride": ctypes.c_int64, "utterance_offset": ctypes.c_int64,
            "sampling_rate": ctypes.c_double, "alpha": ctypes.c_float}
    seen = {(p, t) for _, params in parsed.values() for t, p in params if p in want}
    assert seen == set(want.items())
    for decl in ("int b2d_x(bool flag);", "long double b2d_x(int n);", "int b2d_x(int);", "int b2d_x(const float*, int n);"):
        with pytest.raises(ValueError, match=re.escape(decl)):
            _lib.prototypes(decl, "b2d_")


def test_version_and_error_string(lib):
    assert lib.b2d_version() == 100
    rc = lib.b2d_phase_scan(0, 0, 1, 1, 512, 44100.0, 0, 0, 0, 0)
    assert rc == -1   # B2D_ERR_NULL, before any CUDA call
    assert b"null" in lib.b2d_last_error()
    rc = lib.b2d_phase_scan(16, 0, 0, 1, 512, 44100.0, 0, 16, 16, 0)
    assert rc == -2   # B2D_ERR_SHAPE


def test_argument_errors_do_not_touch_the_device(lib):
    assert lib.b2d_sins_bank(16, 16, 16, 128, 1, 1, 510, 128, 44100.0, 0, 16, 0) == -4      # block % 4
    assert lib.b2d_sins_bank(16, 16, 16, 64, 1, 1, 512, 128, 44100.0, 0, 16, 0) == -2       # stride < H
    assert lib.b2d_ir_build(16, 256, 7, 0, 16, 1, 1, 256, 44100.0, 16, 0) == -4             # unknown mode
    assert lib.b2d_ir_build(16, 256, 2, 0, 16, 1, 1, 256, 44100.0, 16, 0) == -1             # dynamic w/o f0
    assert lib.b2d_ltv_fir(16, 16, 510, 16, 0, 0, 0, 0, 0, 0, 0, 1, 1, 100, 0) == -4        # block % 256
    assert lib.b2d_set_fir_impl(1) == 0                                                      # direct form only:
    assert lib.b2d_ltv_fir(16, 16, 510, 16, 16, 16, 1022, 16, 16, 0, 0, 1, 1, 512, 0) == -4  # unequal taps
    assert lib.b2d_set_fir_impl(0) == 0                                                      # (the FFT kernel takes them)
    assert lib.b2d_ltv_fir(16, 16, 511, 16, 0, 0, 0, 0, 0, 0, 0, 1, 1, 512, 0) == -2         # odd tap count
    assert lib.b2d_set_fir_impl(5) == -4
    assert lib.b2d_ltv_fir(4, 16, 510, 16, 0, 0, 0, 0, 0, 0, 0, 1, 1, 512, 0) == -3         # misaligned x
    # sinusoids + two impulse-response tensors (+ two packed-spectrum tensors when the spectrum variant is selected)
    assert lib.b2d_sins_workspace_bytes(32, 861, 512, 256, 256) == 32 * 861 * 512 * 4 + 2 * 32 * 861 * 510 * 4
    assert lib.b2d_set_sins_impl(3) == 0
    assert lib.b2d_sins_workspace_bytes(32, 861, 512, 256, 256) == 32 * 861 * 512 * 4 + 2 * 32 * 861 * 510 * 4 + 2 * 32 * 861 * 1024 * 4
    up = lambda v: (v + 255) // 256 * 256
    assert lib.b2d_sins_workspace_bytes(2, 10, 256, 256, 256) == up(2 * 10 * 256 * 4) + 2 * up(2 * 10 * 510 * 4)   # block 256: no spectra
    assert lib.b2d_set_sins_impl(0) == 0
    assert lib.b2d_dft_tables_bytes(256) == 2 * 256 * 128 * 4 + 16 * 8 * 128 * 8 * 4   # CUDA-core tables + tensor-core image
    assert lib.b2d_sins_synth(16, 16, 16, 16, 16, 640, 0, 0, 0, 16, 16, 1, 1, 512, 128, 256, 256, 44100.0, 0,
                              16, 16, 16, 256, 10, 0) == -5                                  # workspace too small
    # the control network's kernels (unit2control.cu, linear_attention.cu); p: a non-null, 16-byte aligned address
    p = 16
    for C in (0, 33, 1056):                                                                  # C % 32, C > 1024
        assert lib.b2d_u2c_layernorm(p, p, 4, C, p, p, 1e-5, 0) == -2
    for B, C, groups in ((1, 128, 4), (1, 256, 3), (65536, 256, 4)):                         # C != 256, C % groups, grid.y
        assert lib.b2d_u2c_groupnorm_lrelu(p, B, 8, C, groups, p, p, 1e-5, 0.01, p, 0) == -2
    for B, inner, k in ((1, 256, 29), (1, 100, 31), (65536, 256, 31)):                       # k != 31, inner % 128, grid.z
        assert lib.b2d_u2c_glu_dwconv_silu(p, p, p, p, B, 8, inner, k, 0) == -2
    assert lib.b2d_u2c_softmax_features(p, p, 0, 266, 64, 1, 1e-4, 0) == -2
    assert lib.b2d_u2c_linear_attention(p, p, p, p, 1, 8, 16, 266, 32, 1e-8, 0) == -4         # dim_head != 64
    assert lib.b2d_u2c_linear_attention(p, p, p, p, 1, 8, 16, 273, 64, 1e-8, 0) == -4         # > 272 features
    assert lib.b2d_split_tf32(p + 4, p, p, 8, 0) == -3                                        # misaligned x
    assert lib.b2d_split_tf32(p, p, p, 0, 0) == 0                                             # nothing to do
    assert lib.b2d_u2c_embed(p, p, p, p, p, p, 2, 0, 3, 10, 0) == -2                          # spk_rows not 1 or B


def test_ops_refuse_cpu_tensors():
    import torch
    from ddsp_svc_b200 import ops
    with pytest.raises(ValueError):
        ops.phase_scan(torch.zeros(1, 4, 1), 512, 44100)
