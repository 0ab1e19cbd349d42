"""ctypes binding of libdetzero_b200.so.

include/detzero_b200.h is the one record of the C ABI: every entry point's restype / argtypes and every enum constant are read
from it when this module is imported, so a new entry point is callable as lib().dz_new(...) without an edit here.
There is no CPU fallback: if the library is missing, or a call fails, this raises."""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdetzero_b200.so')
HEADER_PATH = os.path.join(_HERE, '..', 'include', 'detzero_b200.h')

#: the C types a prototype may use, other than pointers (every pointer is a c_void_p)
_CTYPES = {'int': ctypes.c_int, 'size_t': ctypes.c_size_t, 'float': ctypes.c_float, 'double': ctypes.c_double,
           'long long': ctypes.c_longlong, 'unsigned long long': ctypes.c_uint64, 'dz_stream_t': ctypes.c_void_p}


def _ctype(entry, decl):
    """ctypes type of the declaration `decl` ('const float* x', 'size_t n') in the prototype of `entry`"""
    words = decl.replace('*', ' * ').split()
    if '*' in words:
        return ctypes.c_void_p
    if ' '.join(words[:-1]) not in _CTYPES:
        raise ValueError('%s: no ctypes type for %r' % (entry, ' '.join(words)))
    return _CTYPES[' '.join(words[:-1])]


def parse_header(text):
    """C header text -> ({name: (restype, argtypes)} of every dz_* prototype, {name: value} of every enum constant).
    Raises ValueError, naming the entry point, on a prototype it cannot read or a type outside _CTYPES."""
    text = re.sub(r'/\*.*?\*/|//[^\n]*|^[ \t]*#[^\n]*', ' ', text, flags=re.S | re.M)
    consts = {}
    for body in re.findall(r'\benum\s*\{([^}]*)\}', text):
        for item in body.split(','):
            name, value = item.split('=')
            consts[name.strip()] = int(value)
    sigs = {}
    for decl in re.split(r'[;{}]', text):
        found = re.search(r'\b(dz_\w+)\s*\(', decl)
        if not found:
            continue
        name = found.group(1)
        m = re.fullmatch(r'\s*([\w\s*]+?)\s*\b%s\s*\(([^()]*)\)\s*' % name, decl)
        if not m:
            raise ValueError('%s: cannot read the prototype %r' % (name, ' '.join(decl.split())))
        ret, params = ' '.join(m.group(1).split()), m.group(2)
        sigs[name] = (ctypes.c_char_p if ret == 'const char*' else _ctype(name, ret + ' ' + name),
                      [] if params.strip() == 'void' else [_ctype(name, p) for p in params.split(',')])
    return sigs, consts


#: _SIGS: {name: (restype, argtypes)} of every entry point the header declares
with open(HEADER_PATH) as _f:
    _SIGS, _CONSTANTS = parse_header(_f.read())
globals().update(_CONSTANTS)        # DZ_OK, DZ_ERR_*, DZ_F32 .. DZ_BF16X2, DZ_TTA_*, DZ_TTA_MAX_VIEWS, DZ_WBF_MAX_LABELS

MODES = {'fp32': DZ_F32, 'f32': DZ_F32, 'tf32': DZ_TF32, 'bf16': DZ_BF16, 'tf32x3': DZ_TF32X3, 'fp32_tc': DZ_TF32X3,
         'bf16x2': DZ_BF16X2}
#: bf16 operand planes per mode (sparse conv, csrc/spconv_bf16.cu)
PLANES = {DZ_BF16: 1, DZ_BF16X2: 2}

_lib = None


def lib():
    """Load the library (once).  Raises if it has not been built -- the product path never falls back to CPU."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                'detzero_b200: %s is missing. Build it with `python -c "import __graft_entry__ as g; g.build()"` '
                '(nvcc, sm_90a). There is no CPU fallback.' % LIB_PATH)
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)            # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def exported_symbols():
    return sorted(_SIGS)


def check(rc, what=''):
    if rc != 0:
        msg = lib().dz_last_error_string()
        raise RuntimeError('detzero_b200 %s failed (rc=%d): %s' % (what, rc, msg.decode() if msg else ''))


def farr(vals):
    return (ctypes.c_float * len(vals))(*[float(v) for v in vals])


def iarr(vals):
    return (ctypes.c_int * len(vals))(*[int(v) for v in vals])


def darr(vals):
    return (ctypes.c_double * len(vals))(*[float(v) for v in vals])
