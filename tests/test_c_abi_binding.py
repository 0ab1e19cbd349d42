"""CPU tests: the ctypes binding read from include/detzero_b200.h (detzero_b200/_lib.py) -- every declared entry point, one
spot check per row of the C -> ctypes type table, the enum constants, and loud failure on a prototype it cannot bind.
Needs neither a GPU nor the built library."""
import ctypes
import os
import re

import pytest

from detzero_b200 import _lib

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'detzero_b200.h')
V, I, S = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t


def _header():
    with open(HEADER) as f:
        return f.read()


def test_every_declared_entry_point_is_parsed():
    declared = set(re.findall(r'\b(dz_[a-z0-9_]+)\s*\(', _header()))
    assert declared == set(_lib._SIGS) == set(_lib.exported_symbols())
    assert _lib.parse_header(_header())[0] == _lib._SIGS


def test_types_from_the_header():
    sig = _lib._SIGS
    assert sig['dz_scan_ws_bytes'] == (S, [S])
    assert sig['dz_voxelize_hard_batch'][1][0] is V                         # const float* const* points_host
    res, args = sig['dz_refine_inputs']
    assert res is I and len(args) == 35
    assert args[20] is ctypes.c_double and args[23] is ctypes.c_uint64     # enlarge_scale, seed
    assert args[33] is S and args[34] is V                                  # ws_bytes, stream
    assert sig['dz_refine_train_draw'][1][7:9] == [ctypes.c_uint64, ctypes.c_longlong]   # seed, epoch
    assert sig['dz_last_error_string'] == (ctypes.c_char_p, [])
    assert sig['dz_version'] == (I, [])
    assert [i for i, t in enumerate(sig['dz_centerhead_decode'][1]) if t is ctypes.c_float] == [17]     # score_thresh
    assert [i for i, t in enumerate(sig['dz_layernorm_residual'][1]) if t is ctypes.c_float] == [4]     # eps
    assert sig['dz_pm_act'] == (I, [ctypes.c_longlong, I, V, V, V, V])
    assert sig['dz_add'] == (I, [V, V, S, V, V])


def test_enum_constants():
    assert {k: getattr(_lib, k) for k in _lib._CONSTANTS} == {
        'DZ_OK': 0, 'DZ_ERR_ARG': -1, 'DZ_ERR_CUDA': -2, 'DZ_ERR_WORKSPACE': -3, 'DZ_ERR_UNSUPPORTED': -4,
        'DZ_F32': 0, 'DZ_TF32': 1, 'DZ_BF16': 2, 'DZ_TF32X3': 3, 'DZ_BF16X2': 4,
        'DZ_TTA_ORIGINAL': 0, 'DZ_TTA_FLIP_X': 1, 'DZ_TTA_FLIP_Y': 2, 'DZ_TTA_FLIP_XY': 3, 'DZ_TTA_ROT': 4, 'DZ_TTA_SCALE': 5,
        'DZ_TTA_MAX_VIEWS': 32, 'DZ_WBF_MAX_LABELS': 8}
    assert _lib.MODES == {'fp32': 0, 'f32': 0, 'tf32': 1, 'bf16': 2, 'tf32x3': 3, 'fp32_tc': 3, 'bf16x2': 4}
    assert _lib.PLANES == {2: 1, 4: 2}


def test_an_edited_header_binds_as_written():
    proto = 'int dz_add(const float* a, const float* b, size_t n, float* out, dz_stream_t stream);'
    text = _header()
    assert proto in text
    sigs, _ = _lib.parse_header(text.replace(proto, proto.replace('size_t n', 'int n'))
                                + '\nsize_t dz_new(double a, unsigned long long b, const float* const* c);\n')
    assert sigs.pop('dz_add') == (I, [V, V, I, V, V])
    assert sigs.pop('dz_new') == (S, [ctypes.c_double, ctypes.c_uint64, V])
    assert sigs == {k: v for k, v in _lib._SIGS.items() if k != 'dz_add'}


@pytest.mark.parametrize('proto, message', [
    ('int dz_new(int n, uint16_t x, dz_stream_t stream);', "dz_new: no ctypes type for 'uint16_t x'"),
    ('unsigned dz_new(int n);', "dz_new: no ctypes type for 'unsigned dz_new'"),
    ('int dz_new(int);', "dz_new: no ctypes type for 'int'"),
    ('int dz_new(void (*cb)(int));', 'dz_new: cannot read the prototype'),
])
def test_a_prototype_it_cannot_bind_raises(proto, message):
    with pytest.raises(ValueError, match=re.escape(message)):
        _lib.parse_header(_header() + '\n' + proto + '\n')
