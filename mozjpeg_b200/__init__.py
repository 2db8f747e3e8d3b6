"""mozjpeg_b200 -- GPU-native (H100) JPEG encode hot path behind the reference's API.

Python here is plumbing only: it sequences calls into ``libb200jpeg.so`` (the
C-ABI of ``include/b200jpeg.h``; hand-written sm_90a kernels).  There is no
CPU path: importing fails if the library is not built, encoding fails if no
CUDA device is usable.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from . import _abi as A
from ._abi import B200JpegError, Params  # noqa: F401
from .cjpeg import params_from_switches, read_ppm  # noqa: F401

_lib = A.load()          # raises ImportError with build instructions if missing

__all__ = ["Encoder", "Params", "params_from_switches", "read_ppm", "cjpeg", "tj3_params", "B200JpegError"]


class Encoder:
    """One CUDA device + stream + HBM arenas (b200jpeg_encoder)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        A.check(_lib.b200jpeg_encoder_create(C.byref(self._h), device), "encoder_create")

    def close(self) -> None:
        if self._h:
            _lib.b200jpeg_encoder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int) -> None:
        """Launch on a caller-owned stream (e.g. torch.cuda.current_stream().cuda_stream)."""
        A.check(_lib.b200jpeg_encoder_set_stream(self._h, C.c_void_p(cuda_stream)), "set_stream")

    def set_chunk_images(self, n: int) -> None:
        """Images per pipeline chunk (0 = automatic)."""
        A.check(_lib.b200jpeg_encoder_set_chunk_images(self._h, n), "set_chunk_images")

    def chunk_images(self) -> int:
        """Images per chunk (= per kernel launch) of the last batch."""
        return int(_lib.b200jpeg_last_chunk_images(self._h))

    def set_streams(self, n: int) -> None:
        """Compute streams consecutive chunks alternate between (1 or 2)."""
        A.check(_lib.b200jpeg_encoder_set_streams(self._h, n), "set_streams")

    # -- batch API -------------------------------------------------------
    def encode_batch(self, p: Params, images: np.ndarray) -> List[bytes]:
        """images: (N, H, W, C) or (N, H, W) host array -> N JPEG files (uint8, or uint16
        holding 12-bit samples when p.data_precision == 12, like J12SAMPLE rows).
        Host->device staging and device->host read-back happen inside."""
        a = np.ascontiguousarray(images, dtype=np.uint16 if p.data_precision == 12 else np.uint8)
        if a.ndim == 3 and p.input_components == 1:
            a = a[..., None]
        n, h, w, c = a.shape
        if (w, h, c) != (p.image_width, p.image_height, p.input_components):
            raise ValueError("array shape does not match params")
        A.check(_lib.b200jpeg_encode_batch(self._h, C.byref(p), a.ctypes.data, 0, a.strides[1], a.strides[0], n), "encode_batch")
        return [self.get_output(i) for i in range(n)]

    def encode_batch_raw(self, p: Params, planes: Sequence[np.ndarray]) -> List[bytes]:
        """Raw-data input (jpeg_write_raw_data): planes[ci] is an (N, rows, cols) uint8 array holding
        the converted, downsampled samples of component ci (at least hib*8 x wib*8 per image)."""
        arrs = [np.ascontiguousarray(a, dtype=np.uint8) for a in planes]
        n = arrs[0].shape[0]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        pitch = (C.c_size_t * len(arrs))(*[a.strides[1] for a in arrs])
        stride = (C.c_size_t * len(arrs))(*[a.strides[0] for a in arrs])
        A.check(_lib.b200jpeg_encode_batch_raw(self._h, C.byref(p), ptrs, 0, pitch, stride, n), "encode_batch_raw")
        return [self.get_output(i) for i in range(n)]

    def encode_batch_coefs(self, p: Params, planes: Sequence[np.ndarray]) -> List[bytes]:
        """Coefficient-domain input (jpeg_write_coefficients): planes[ci] is an (N, hib, wib, 64) int16 array of
        quantized coefficients in natural order (libjpeg JBLOCKs)."""
        arrs = [np.ascontiguousarray(a, dtype=np.int16) for a in planes]
        n = arrs[0].shape[0]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        pitch = (C.c_size_t * len(arrs))(*[a.strides[1] // 128 for a in arrs])
        stride = (C.c_size_t * len(arrs))(*[a.strides[0] // 128 for a in arrs])
        A.check(_lib.b200jpeg_encode_batch_coefs(self._h, C.byref(p), ptrs, 0, pitch, stride, n), "encode_batch_coefs")
        return [self.get_output(i) for i in range(n)]

    def encode_batch_ptr(self, p: Params, ptr: int, on_device: bool, row_pitch: int, image_stride: int, n: int,
                         device_only: bool = False) -> None:
        """Raw-pointer form (device tensors, pinned host buffers)."""
        if device_only:
            A.check(_lib.b200jpeg_encode_batch_device_only(self._h, C.byref(p), ptr, row_pitch, image_stride, n), "encode_batch_device_only")
        else:
            A.check(_lib.b200jpeg_encode_batch(self._h, C.byref(p), ptr, int(on_device), row_pitch, image_stride, n), "encode_batch")

    def get_output(self, i: int) -> bytes:
        d = C.POINTER(C.c_uint8)(); n = C.c_size_t(0)
        A.check(_lib.b200jpeg_get_output(self._h, i, C.byref(d), C.byref(n)), "get_output")
        return C.string_at(d, n.value)

    def output_size(self, i: int) -> int:
        n = C.c_size_t(0)
        A.check(_lib.b200jpeg_get_output(self._h, i, None, C.byref(n)), "get_output")
        return n.value

    # -- streaming shim (jpeg_start_compress / write_scanlines / finish) ---
    def start_compress(self, p: Params) -> None:
        A.check(_lib.b200jpeg_start_compress(self._h, C.byref(p)), "start_compress")

    def write_scanlines(self, rows: np.ndarray) -> int:
        r = np.ascontiguousarray(rows, dtype=np.uint8)
        if r.ndim == 2:
            r = r[None]
        ptrs = (C.POINTER(C.c_uint8) * r.shape[0])()
        for i in range(r.shape[0]):
            ptrs[i] = r[i].ctypes.data_as(C.POINTER(C.c_uint8))
        return A.check(_lib.b200jpeg_write_scanlines(self._h, ptrs, r.shape[0]), "write_scanlines")

    def finish_compress(self) -> bytes:
        d = C.POINTER(C.c_uint8)(); n = C.c_size_t(0)
        A.check(_lib.b200jpeg_finish_compress(self._h, C.byref(d), C.byref(n)), "finish_compress")
        return C.string_at(d, n.value)

    # -- introspection -----------------------------------------------------
    def kernel_launches(self) -> int:
        return int(_lib.b200jpeg_kernel_launches(self._h))

    def last_scan_bytes(self) -> int:
        return int(_lib.b200jpeg_last_scan_bytes(self._h))

    def stage_times(self) -> dict:
        names = (C.c_char_p * 32)(); ms = (C.c_float * 32)()
        k = _lib.b200jpeg_last_stage_times(self._h, names, ms, 32)
        return {names[i].decode(): float(ms[i]) for i in range(k)}

    def debug_coefs(self, image: int, component: int, plane: int = 0) -> np.ndarray:
        """[hpad][wpad][64] int16, natural order (plane 0 final, 1 raw DCT, 2 plain-quantized)."""
        wib = C.c_int(0); hib = C.c_int(0)
        nb = A.check(_lib.b200jpeg_debug_get_coefs(self._h, image, component, plane, None, 0, C.byref(wib), C.byref(hib)), "debug_get_coefs")
        out = np.zeros((hib.value, wib.value, 64), dtype=np.int16)
        A.check(_lib.b200jpeg_debug_get_coefs(self._h, image, component, plane, out.ctypes.data_as(C.POINTER(C.c_int16)), nb, None, None), "debug_get_coefs")
        return out

    def debug_huff(self, image: int, scan: int, is_ac: bool, tbl_no: int):
        h = A.HuffTbl()
        A.check(_lib.b200jpeg_debug_get_huff(self._h, image, scan, int(is_ac), tbl_no, C.byref(h)), "debug_get_huff")
        bits = tuple(h.bits); n = sum(bits[1:])
        return bits, tuple(h.huffval)[:n]


def cjpeg(switches: Sequence[str], ppm: bytes, encoder: Optional[Encoder] = None) -> bytes:
    """``cjpeg <switches> file.ppm`` on the device path: PPM/PGM bytes -> JPEG bytes."""
    w, h, nc, data = read_ppm(ppm)
    p = params_from_switches(switches, w, h, nc)
    img = np.frombuffer(data, dtype=np.uint8).reshape(1, h, w, nc)
    enc = encoder or Encoder(0)
    try:
        return enc.encode_batch(p, img)[0]
    finally:
        if encoder is None:
            enc.close()


def tj3_params(width: int, height: int, quality: int = 75, subsamp: str = "420", optimize: bool = False,
               progressive: bool = False, gray_input: bool = False) -> Params:
    """The parameter block tj3Compress8 builds (turbojpeg.c:330-397
    setCompDefaults): JCP_FASTEST, quality via jpeg_set_quality(.., TRUE),
    YCbCr (or grayscale) with the luma sampling factors of TJSAMP_*."""
    p = Params()
    p.in_color_space = A.CS_GRAYSCALE if gray_input else A.CS_RGB
    p.input_components = 1 if gray_input else 3
    p.data_precision = 8
    p.image_width, p.image_height = width, height
    _lib.b200jpeg_set_defaults(C.byref(p), A.PROFILE_FASTEST)
    p.image_width, p.image_height = width, height
    p.optimize_coding = int(optimize)
    _lib.b200jpeg_set_quality(C.byref(p), quality, 1)
    gray = gray_input or subsamp == "gray"
    A.check(_lib.b200jpeg_set_colorspace(C.byref(p), A.CS_GRAYSCALE if gray else A.CS_YCbCr), "set_colorspace")
    if progressive:
        A.check(_lib.b200jpeg_simple_progression(C.byref(p)), "simple_progression")
    hv = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2), "411": (4, 1), "441": (1, 4), "gray": (1, 1)}[subsamp]
    p.comp_info[0].h_samp_factor, p.comp_info[0].v_samp_factor = hv
    for ci in range(1, p.num_components):
        p.comp_info[ci].h_samp_factor = p.comp_info[ci].v_samp_factor = 1
    return p
