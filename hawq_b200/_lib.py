"""ctypes binding of libhawq_b200.so (C ABI: include/hawq_b200.h).

The library is built in-tree by ``hawq_b200.build.build_library`` (nvcc, sm_90a).  There is NO fallback: if the
shared object is missing or cannot be loaded, every product entry point raises ``HawqLibraryError``.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libhawq_b200.so")


class HawqLibraryError(RuntimeError):
    pass


class HawqError(RuntimeError):
    """A C-ABI call returned a negative hawq_status."""

    def __init__(self, code, msg):
        super().__init__("hawq_b200 error %d: %s" % (code, msg))
        self.code = code


class hawq_chan(C.Structure):
    _fields_ = [("bias", C.c_int32), ("m", C.c_uint32), ("e", C.c_int32), ("reserved", C.c_int32)]


class hawq_conv_desc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("N", "H", "W", "Cin", "Cout", "kh", "kw", "stride", "pad", "a_bits", "w_layout")]


class hawq_epilogue_desc(C.Structure):
    _fields_ = [("mode", C.c_int32), ("relu", C.c_int32), ("out_bits", C.c_int32), ("clamp_lo", C.c_int32),
                ("clamp_hi", C.c_int32), ("res_kind", C.c_int32), ("res_bits", C.c_int32), ("res_m", C.c_uint32),
                ("res_e", C.c_int32), ("y_bits", C.c_int32), ("low_bits", C.c_int32), ("low_m", C.c_uint32),
                ("low_e", C.c_int32), ("low_lo", C.c_int32), ("low_hi", C.c_int32), ("cout_store", C.c_int32),
                ("flags", C.c_int32)]


EPI_REQUANT, EPI_RESIDUAL, EPI_RAW_I32, EPI_DEQUANT_F32 = 0, 1, 2, 3
FLAG_RESIDUAL_OVERFLOW = 1
FLAG_BAD_RATIO = 2
FLAG_REQUANT_OVERFLOW = 4
EP_RATIOS_LE_ONE = 1
EP_RATIOS_LE_2P20 = 2
ERR_BAD_ARG, ERR_UNSUPPORTED, ERR_CUDA, ERR_RESULT_INVALID = -1, -2, -3, -4   # hawq_status


class hawq_engine_info(C.Structure):
    _fields_ = [("input_dtype", C.c_int32), ("residual_bits", C.c_int32), ("input_shape", C.c_int64 * 4), ("input_bytes", C.c_int64),
                ("output_shape", C.c_int64 * 2), ("arena_bytes", C.c_int64), ("constant_bytes", C.c_int64), ("launches", C.c_int64 * 3),
                ("fallbacks", C.c_int64)]


# enum hawq_engine_entry: the entry id of each entry point in a plan file is its index here
ENGINE_ENTRIES = ("hawq_conv2d", "hawq_conv2d_dual", "hawq_linear_i8", "hawq_stem_conv_i8", "hawq_stem_pool_i8", "hawq_dwconv3x3",
                  "hawq_stem3x3_i8", "hawq_maxpool_requant", "hawq_avgpool_requant", "hawq_quantize_input_f32", "hawq_quantize_input_u8",
                  "hawq_resize_crop_quantize_u8", "hawq_requant", "hawq_add_requant", "hawq_dequant_f32", "hawq_pack_i4", "hawq_unpack_i4")
ENGINE_FORMAT = 1

_vp, _i32, _i64, _u32, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_float
_conv_args = [_vp, C.POINTER(hawq_conv_desc), C.POINTER(hawq_epilogue_desc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]

# every symbol include/hawq_b200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "hawq_abi_version": (_i32, []),
    "hawq_last_error": (C.c_char_p, []),
    "hawq_create": (_i32, [_i32, C.POINTER(_vp)]),
    "hawq_destroy": (_i32, [_vp]),
    "hawq_sm_count": (_i32, [_vp]),
    "hawq_reset_status": (_i32, [_vp, _vp]),
    "hawq_get_status": (_i32, [_vp, _vp, C.POINTER(_i32)]),
    "hawq_copy_status": (_i32, [_vp, _vp, _vp]),
    "hawq_conv2d": (_i32, _conv_args),
    "hawq_conv2d_i8": (_i32, _conv_args),
    "hawq_conv2d_i4": (_i32, _conv_args),
    "hawq_conv2d_dual": (_i32, [_vp, C.POINTER(hawq_conv_desc), C.POINTER(hawq_epilogue_desc), _vp, _vp, _vp,
                                C.POINTER(hawq_conv_desc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "hawq_linear_i8": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "hawq_stem_conv_i8": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "hawq_stem_pool_i8": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _i32, _u32, _i32, _i32, _i32, _vp, _vp]),
    "hawq_dwconv3x3": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "hawq_stem3x3_i8": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _u32, _i32, _i32, _i32, _vp, _vp]),
    "hawq_maxpool_requant": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _i32, _vp, _i32, _u32, _i32, _i32, _i32, _vp, _vp]),
    "hawq_avgpool_requant": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _u32, _i32, _i32, _i32, _vp, _vp]),
    "hawq_quantize_input_f32": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _f32, _i32, _i32, _vp, _vp]),
    "hawq_quantize_input_u8": (_i32, [_vp, _i32, _i32, _i32, _vp, C.POINTER(_f32), C.POINTER(_f32), _f32, _i32, _i32, _vp, _vp]),
    "hawq_resize_crop_quantize_u8": (_i32, [_vp, _i32, _vp, _i64, _vp, _i32, _i32, _i32, C.POINTER(_f32), C.POINTER(_f32), _f32, _i32,
                                            _i32, _vp, _vp]),
    "hawq_requant": (_i32, [_vp, _i64, _i32, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "hawq_add_requant": (_i32, [_vp, _i64, _i32, _vp, _vp, C.POINTER(hawq_epilogue_desc), _vp, _vp, _vp, _vp, _vp]),
    "hawq_dequant_f32": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _f32, _vp, _vp]),
    "hawq_pack_i4": (_i32, [_vp, _i64, _vp, _vp, _vp]),
    "hawq_unpack_i4": (_i32, [_vp, _i64, _vp, _vp, _vp]),
    "hawq_dyadic": (_i32, [C.c_double, C.POINTER(_u32), C.POINTER(_i32)]),
    "hawq_rhe_requant_host": (_i64, [_i32, _u32, _i32]),
    "hawq_permute_weights_for_i4": (_i32, [_vp, _i64, _i32]),
    "hawq_retile_weights": (_i32, [_vp, _vp, _i32, _i64, _vp, _vp]),
    "hawq_debug_kernel_count": (_i64, [_i32]),
    "hawq_workspace_bytes": (_i64, [C.POINTER(hawq_conv_desc), C.POINTER(hawq_epilogue_desc)]),
    "hawq_engine_check": (_i32, [_vp, _i64, C.POINTER(hawq_engine_info)]),
    "hawq_engine_load": (_i32, [_i32, _vp, _i64, C.POINTER(_vp)]),
    "hawq_engine_destroy": (_i32, [_vp]),
    "hawq_engine_input": (_vp, [_vp]),
    "hawq_engine_output": (_vp, [_vp]),
    "hawq_engine_get_info": (_i32, [_vp, C.POINTER(hawq_engine_info)]),
    "hawq_engine_enqueue": (_i32, [_vp, _vp]),
    "hawq_engine_status": (_i32, [_vp, C.POINTER(_i32)]),
    "hawq_engine_run": (_i32, [_vp, _vp, C.POINTER(_i32)]),
}

_lib = None


def load():
    """Load libhawq_b200.so and bind every declared symbol (raises HawqLibraryError on any problem)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise HawqLibraryError(
            "%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). hawq_b200 has no CPU or PyTorch fallback." % LIB_PATH)
    try:
        lib = C.CDLL(LIB_PATH)
    except OSError as e:
        raise HawqLibraryError("cannot load %s: %s" % (LIB_PATH, e))
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise HawqLibraryError("%s does not export %s (stale build?)" % (LIB_PATH, name))
        fn.restype = res
        fn.argtypes = args
    if lib.hawq_abi_version() != 1:
        raise HawqLibraryError("ABI version mismatch: library %d, binding 1" % lib.hawq_abi_version())
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise HawqError(rc, load().hawq_last_error().decode("utf-8", "replace"))


def dyadic(ratio):
    """(m, e) of batch_frexp for one ratio, via the library's host helper."""
    m, e = _u32(), _i32()
    check(load().hawq_dyadic(float(ratio), C.byref(m), C.byref(e)))
    return int(m.value), int(e.value)
