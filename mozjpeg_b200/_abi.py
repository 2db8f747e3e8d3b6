"""ctypes binding of libb200jpeg.so (the C-ABI in include/b200jpeg.h).

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).
There is no fallback: if the shared object is missing the import fails loudly,
and the encode entry points fail with B200JPEG_ERR_NO_DEVICE when no CUDA
device is usable.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200jpeg.so")
if os.environ.get("B200JPEG_LIB_VARIANT"):            # development aid (tools/build_variant.sh): A/B builds of the kernels
    LIB_PATH = os.path.join(_HERE, "variants", "libb200jpeg_%s.so" % os.environ["B200JPEG_LIB_VARIANT"])

MAX_COMPONENTS = 4
NUM_QUANT_TBLS = 4
NUM_HUFF_TBLS = 4
MAX_SCANS = 64

CS_UNKNOWN, CS_GRAYSCALE, CS_RGB, CS_YCbCr, CS_CMYK, CS_YCCK = 0, 1, 2, 3, 4, 5
# input pixel orders of the RGB family (J_COLOR_SPACE values, jpeglib.h:243-266): name -> (value, samples per pixel, R, G, B offsets)
CS_EXT = {"EXT_RGB": (6, 3, 0, 1, 2), "EXT_RGBX": (7, 4, 0, 1, 2), "EXT_BGR": (8, 3, 2, 1, 0), "EXT_BGRX": (9, 4, 2, 1, 0),
          "EXT_XBGR": (10, 4, 3, 2, 1), "EXT_XRGB": (11, 4, 1, 2, 3), "EXT_RGBA": (12, 4, 0, 1, 2), "EXT_BGRA": (13, 4, 2, 1, 0),
          "EXT_ABGR": (14, 4, 3, 2, 1), "EXT_ARGB": (15, 4, 1, 2, 3)}
DCT_ISLOW, DCT_IFAST, DCT_FLOAT = 0, 1, 2
PROFILE_MAX_COMPRESSION = 0x5D083AAD
PROFILE_FASTEST = 0x2AEA5CB4

OK = 0
ERR_PARAM, ERR_UNSUPPORTED, ERR_NO_DEVICE, ERR_CUDA, ERR_BUFFER, ERR_BAD_DCT_COEF, ERR_STATE = -1, -2, -3, -4, -5, -6, -7


class ScanInfo(C.Structure):
    _fields_ = [("comps_in_scan", C.c_int), ("component_index", C.c_int * MAX_COMPONENTS),
                ("Ss", C.c_int), ("Se", C.c_int), ("Ah", C.c_int), ("Al", C.c_int)]


class ComponentInfo(C.Structure):
    _fields_ = [("component_id", C.c_int), ("h_samp_factor", C.c_int), ("v_samp_factor", C.c_int),
                ("quant_tbl_no", C.c_int), ("dc_tbl_no", C.c_int), ("ac_tbl_no", C.c_int)]


class HuffTbl(C.Structure):
    _fields_ = [("bits", C.c_uint8 * 17), ("huffval", C.c_uint8 * 256), ("present", C.c_int)]


class Params(C.Structure):
    """b200jpeg_params: the encoder-relevant fields of jpeg_compress_struct +
    jpeg_comp_master under the reference's names (jpeglib.h:388-561,
    jpegint.h:93-135)."""
    _fields_ = [
        ("image_width", C.c_int), ("image_height", C.c_int), ("input_components", C.c_int),
        ("in_color_space", C.c_int), ("data_precision", C.c_int),
        ("jpeg_color_space", C.c_int), ("num_components", C.c_int),
        ("comp_info", ComponentInfo * MAX_COMPONENTS),
        ("quant_tbl", (C.c_uint16 * 64) * NUM_QUANT_TBLS),
        ("quant_tbl_present", C.c_int * NUM_QUANT_TBLS),
        ("dc_huff_tbl", HuffTbl * NUM_HUFF_TBLS), ("ac_huff_tbl", HuffTbl * NUM_HUFF_TBLS),
        ("num_scans", C.c_int), ("scan_info", ScanInfo * MAX_SCANS),
        ("optimize_coding", C.c_int), ("dct_method", C.c_int),
        ("restart_interval", C.c_int), ("restart_in_rows", C.c_int), ("smoothing_factor", C.c_int),
        ("write_JFIF_header", C.c_int), ("JFIF_major_version", C.c_int), ("JFIF_minor_version", C.c_int),
        ("density_unit", C.c_int), ("X_density", C.c_int), ("Y_density", C.c_int),
        ("write_Adobe_marker", C.c_int),
        ("compress_profile", C.c_int), ("optimize_scans", C.c_int),
        ("trellis_quant", C.c_int), ("trellis_quant_dc", C.c_int), ("trellis_eob_opt", C.c_int),
        ("use_lambda_weight_tbl", C.c_int), ("use_scans_in_trellis", C.c_int), ("trellis_q_opt", C.c_int),
        ("overshoot_deringing", C.c_int), ("trellis_freq_split", C.c_int), ("trellis_num_loops", C.c_int),
        ("quant_tbl_master_idx", C.c_int), ("dc_scan_opt_mode", C.c_int),
        ("lambda_log_scale1", C.c_float), ("lambda_log_scale2", C.c_float),
        ("trellis_delta_dc_weight", C.c_float),
        ("q_scale_factor", C.c_int * NUM_QUANT_TBLS),
    ]

    def copy(self) -> "Params":
        q = Params()
        C.memmove(C.byref(q), C.byref(self), C.sizeof(Params))
        return q


# every symbol include/b200jpeg.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "b200jpeg_set_defaults", "b200jpeg_default_colorspace", "b200jpeg_set_colorspace",
    "b200jpeg_quality_scaling", "b200jpeg_float_quality_scaling", "b200jpeg_add_quant_table",
    "b200jpeg_set_linear_quality", "b200jpeg_set_quality", "b200jpeg_default_qtables",
    "b200jpeg_simple_progression", "b200jpeg_enable_lossless", "b200jpeg_std_huff_tables", "b200jpeg_std_quant_tbl",
    "b200jpeg_validate", "b200jpeg_total_passes",
    "b200jpeg_encoder_create", "b200jpeg_encoder_destroy", "b200jpeg_encoder_set_stream", "b200jpeg_encoder_set_chunk_images", "b200jpeg_last_chunk_images", "b200jpeg_encoder_set_streams", "b200jpeg_encode_batch",
    "b200jpeg_encode_batch_device_only", "b200jpeg_encode_batch_raw", "b200jpeg_encode_batch_coefs",
    "b200jpeg_encode_batch_qtables", "b200jpeg_encode_batch_raw_qtables", "b200jpeg_encode_batch_coefs_qtables", "b200jpeg_get_output", "b200jpeg_last_scan_bytes",
    "b200jpeg_kernel_launches", "b200jpeg_last_stage_times", "b200jpeg_debug_get_coefs",
    "b200jpeg_debug_get_huff", "b200jpeg_start_compress", "b200jpeg_write_scanlines",
    "b200jpeg_finish_compress", "b200jpeg_last_error", "b200jpeg_version",
]

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the CUDA extension has not been built. "
            "Run `python -c 'import __graft_entry__ as g; g.build()'` at the repo root. "
            "There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    P = C.POINTER(Params)
    lib.b200jpeg_set_defaults.argtypes = [P, C.c_int]; lib.b200jpeg_set_defaults.restype = None
    lib.b200jpeg_default_colorspace.argtypes = [P]; lib.b200jpeg_default_colorspace.restype = C.c_int
    lib.b200jpeg_set_colorspace.argtypes = [P, C.c_int]; lib.b200jpeg_set_colorspace.restype = C.c_int
    lib.b200jpeg_quality_scaling.argtypes = [C.c_int]; lib.b200jpeg_quality_scaling.restype = C.c_int
    lib.b200jpeg_float_quality_scaling.argtypes = [C.c_float]; lib.b200jpeg_float_quality_scaling.restype = C.c_float
    lib.b200jpeg_add_quant_table.argtypes = [P, C.c_int, C.POINTER(C.c_uint), C.c_int, C.c_int]; lib.b200jpeg_add_quant_table.restype = C.c_int
    lib.b200jpeg_set_linear_quality.argtypes = [P, C.c_int, C.c_int]; lib.b200jpeg_set_linear_quality.restype = None
    lib.b200jpeg_set_quality.argtypes = [P, C.c_int, C.c_int]; lib.b200jpeg_set_quality.restype = None
    lib.b200jpeg_default_qtables.argtypes = [P, C.c_int]; lib.b200jpeg_default_qtables.restype = None
    lib.b200jpeg_simple_progression.argtypes = [P]; lib.b200jpeg_simple_progression.restype = C.c_int
    lib.b200jpeg_enable_lossless.argtypes = [P, C.c_int, C.c_int]; lib.b200jpeg_enable_lossless.restype = C.c_int
    lib.b200jpeg_std_huff_tables.argtypes = [P]; lib.b200jpeg_std_huff_tables.restype = None
    lib.b200jpeg_std_quant_tbl.argtypes = [C.c_int, C.c_int]; lib.b200jpeg_std_quant_tbl.restype = C.POINTER(C.c_uint)
    lib.b200jpeg_validate.argtypes = [P]; lib.b200jpeg_validate.restype = C.c_int
    lib.b200jpeg_total_passes.argtypes = [P]; lib.b200jpeg_total_passes.restype = C.c_int
    lib.b200jpeg_encoder_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]; lib.b200jpeg_encoder_create.restype = C.c_int
    lib.b200jpeg_encoder_destroy.argtypes = [C.c_void_p]; lib.b200jpeg_encoder_destroy.restype = None
    lib.b200jpeg_encoder_set_stream.argtypes = [C.c_void_p, C.c_void_p]; lib.b200jpeg_encoder_set_stream.restype = C.c_int
    lib.b200jpeg_encoder_set_chunk_images.argtypes = [C.c_void_p, C.c_int]; lib.b200jpeg_encoder_set_chunk_images.restype = C.c_int
    lib.b200jpeg_last_chunk_images.argtypes = [C.c_void_p]; lib.b200jpeg_last_chunk_images.restype = C.c_int
    lib.b200jpeg_encoder_set_streams.argtypes = [C.c_void_p, C.c_int]; lib.b200jpeg_encoder_set_streams.restype = C.c_int
    lib.b200jpeg_encode_batch.argtypes = [C.c_void_p, P, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_int]; lib.b200jpeg_encode_batch.restype = C.c_int
    lib.b200jpeg_encode_batch_raw.argtypes = [C.c_void_p, P, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_int]; lib.b200jpeg_encode_batch_raw.restype = C.c_int
    lib.b200jpeg_encode_batch_coefs.argtypes = [C.c_void_p, P, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_int]; lib.b200jpeg_encode_batch_coefs.restype = C.c_int
    Q = C.POINTER(C.c_uint16)
    lib.b200jpeg_encode_batch_qtables.argtypes = [C.c_void_p, P, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, Q, C.c_int]; lib.b200jpeg_encode_batch_qtables.restype = C.c_int
    lib.b200jpeg_encode_batch_raw_qtables.argtypes = [C.c_void_p, P, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), Q, C.c_int]; lib.b200jpeg_encode_batch_raw_qtables.restype = C.c_int
    lib.b200jpeg_encode_batch_coefs_qtables.argtypes = [C.c_void_p, P, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), Q, C.c_int]; lib.b200jpeg_encode_batch_coefs_qtables.restype = C.c_int
    lib.b200jpeg_encode_batch_device_only.argtypes = [C.c_void_p, P, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int]; lib.b200jpeg_encode_batch_device_only.restype = C.c_int
    lib.b200jpeg_get_output.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]; lib.b200jpeg_get_output.restype = C.c_int
    lib.b200jpeg_last_scan_bytes.argtypes = [C.c_void_p]; lib.b200jpeg_last_scan_bytes.restype = C.c_size_t
    lib.b200jpeg_kernel_launches.argtypes = [C.c_void_p]; lib.b200jpeg_kernel_launches.restype = C.c_ulonglong
    lib.b200jpeg_last_stage_times.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.c_int]; lib.b200jpeg_last_stage_times.restype = C.c_int
    lib.b200jpeg_debug_get_coefs.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int16), C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]; lib.b200jpeg_debug_get_coefs.restype = C.c_long
    lib.b200jpeg_debug_get_huff.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(HuffTbl)]; lib.b200jpeg_debug_get_huff.restype = C.c_int
    lib.b200jpeg_start_compress.argtypes = [C.c_void_p, P]; lib.b200jpeg_start_compress.restype = C.c_int
    lib.b200jpeg_write_scanlines.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint8)), C.c_int]; lib.b200jpeg_write_scanlines.restype = C.c_int
    lib.b200jpeg_finish_compress.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]; lib.b200jpeg_finish_compress.restype = C.c_int
    lib.b200jpeg_last_error.argtypes = []; lib.b200jpeg_last_error.restype = C.c_char_p
    lib.b200jpeg_version.argtypes = []; lib.b200jpeg_version.restype = C.c_char_p
    _lib = lib
    return lib


class B200JpegError(RuntimeError):
    def __init__(self, code: int, where: str):
        msg = load().b200jpeg_last_error().decode("utf-8", "replace")
        super().__init__(f"{where}: error {code}: {msg}")
        self.code = code


def check(code: int, where: str) -> int:
    if code < 0:
        raise B200JpegError(code, where)
    return code
