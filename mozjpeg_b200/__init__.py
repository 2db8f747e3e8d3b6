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
from .cjpeg import params_from_switches, pnm_samples, read_pnm, read_ppm  # noqa: F401

_lib = A.load()          # raises ImportError with build instructions if missing

__all__ = ["Encoder", "Params", "params_from_switches", "read_ppm", "cjpeg", "tj3_params", "quality_tables", "B200JpegError"]


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
    # qtables (all three forms): None, or an (N, 4, 64) uint16 array of per-image quantization tables in natural order
    # (the slots p.quant_tbl_present names are read); image i is then written with its own tables.  Input holding ONE
    # image with N table sets is encoded N times from the same pixels (image stride 0, staged once): a quality ladder.
    @staticmethod
    def _qtables(qtables, n: int):
        a = np.asarray(qtables)
        # the conversion to uint16 must not change a value (65537 would become 1 and pass the library's 1..32767 check)
        if a.dtype.kind not in "iu" or (a.size and (a.min() < 0 or a.max() > 0xFFFF)):
            raise ValueError("qtables must hold integers in 0..65535 (the library accepts 1..32767)")
        q = np.ascontiguousarray(a, dtype=np.uint16)
        if q.ndim != 3 or q.shape[1:] != (A.NUM_QUANT_TBLS, 64):
            raise ValueError("qtables must have shape (N, 4, 64)")
        if n != 1 and q.shape[0] != n:
            raise ValueError(f"qtables holds {q.shape[0]} table sets for {n} images")
        return q, q.shape[0], n == 1 and q.shape[0] != 1

    def encode_batch(self, p: Params, images: np.ndarray, qtables: Optional[np.ndarray] = None) -> List[bytes]:
        """images: (N, H, W, C) or (N, H, W) host array -> N JPEG files (uint8, or uint16
        holding 12- or 16-bit samples when p.data_precision is 12 or 16, like J12SAMPLE / J16SAMPLE rows).
        Host->device staging and device->host read-back happen inside."""
        a = np.ascontiguousarray(images, dtype=np.uint16 if p.data_precision > 8 else np.uint8)
        if a.ndim == 3 and p.input_components == 1:
            a = a[..., None]
        n, h, w, c = a.shape
        if (w, h, c) != (p.image_width, p.image_height, p.input_components):
            raise ValueError("array shape does not match params")
        if qtables is None:
            A.check(_lib.b200jpeg_encode_batch(self._h, C.byref(p), a.ctypes.data, 0, a.strides[1], a.strides[0], n), "encode_batch")
        else:
            q, n, shared = self._qtables(qtables, n)
            A.check(_lib.b200jpeg_encode_batch_qtables(self._h, C.byref(p), a.ctypes.data, 0, a.strides[1], 0 if shared else a.strides[0],
                                                       q.ctypes.data_as(C.POINTER(C.c_uint16)), n), "encode_batch_qtables")
        return [self.get_output(i) for i in range(n)]

    def encode_batch_raw(self, p: Params, planes: Sequence[np.ndarray], qtables: Optional[np.ndarray] = None) -> List[bytes]:
        """Raw-data input (jpeg_write_raw_data): planes[ci] is an (N, rows, cols) uint8 array holding
        the converted, downsampled samples of component ci (at least hib*8 x wib*8 per image)."""
        arrs = [np.ascontiguousarray(a, dtype=np.uint8) for a in planes]
        n = arrs[0].shape[0]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        pitch = (C.c_size_t * len(arrs))(*[a.strides[1] for a in arrs])
        if qtables is None:
            stride = (C.c_size_t * len(arrs))(*[a.strides[0] for a in arrs])
            A.check(_lib.b200jpeg_encode_batch_raw(self._h, C.byref(p), ptrs, 0, pitch, stride, n), "encode_batch_raw")
        else:
            q, n, shared = self._qtables(qtables, n)
            stride = (C.c_size_t * len(arrs))(*[0 if shared else a.strides[0] for a in arrs])
            A.check(_lib.b200jpeg_encode_batch_raw_qtables(self._h, C.byref(p), ptrs, 0, pitch, stride, q.ctypes.data_as(C.POINTER(C.c_uint16)), n),
                    "encode_batch_raw_qtables")
        return [self.get_output(i) for i in range(n)]

    def encode_batch_coefs(self, p: Params, planes: Sequence[np.ndarray], qtables: Optional[np.ndarray] = None) -> List[bytes]:
        """Coefficient-domain input (jpeg_write_coefficients): planes[ci] is an (N, hib, wib, 64) int16 array of
        quantized coefficients in natural order (libjpeg JBLOCKs)."""
        arrs = [np.ascontiguousarray(a, dtype=np.int16) for a in planes]
        n = arrs[0].shape[0]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        pitch = (C.c_size_t * len(arrs))(*[a.strides[1] // 128 for a in arrs])
        if qtables is None:
            stride = (C.c_size_t * len(arrs))(*[a.strides[0] // 128 for a in arrs])
            A.check(_lib.b200jpeg_encode_batch_coefs(self._h, C.byref(p), ptrs, 0, pitch, stride, n), "encode_batch_coefs")
        else:
            q, n, shared = self._qtables(qtables, n)
            stride = (C.c_size_t * len(arrs))(*[0 if shared else a.strides[0] // 128 for a in arrs])
            A.check(_lib.b200jpeg_encode_batch_coefs_qtables(self._h, C.byref(p), ptrs, 0, pitch, stride, q.ctypes.data_as(C.POINTER(C.c_uint16)), n),
                    "encode_batch_coefs_qtables")
        return [self.get_output(i) for i in range(n)]

    def encode_batch_qtables_ptr(self, p: Params, ptr: int, on_device: bool, row_pitch: int, image_stride: int,
                                 qtables: np.ndarray) -> None:
        """Raw-pointer form of encode_batch with per-image tables (device tensors, pinned host buffers); one image per
        table set, image_stride 0 = every image reads the same pixels."""
        q, n, _ = self._qtables(qtables, len(qtables))
        A.check(_lib.b200jpeg_encode_batch_qtables(self._h, C.byref(p), ptr, int(on_device), row_pitch, image_stride,
                                                   q.ctypes.data_as(C.POINTER(C.c_uint16)), n), "encode_batch_qtables")

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
        """rows: (n, W, C) or one (W, C) row of uint8 samples, or of uint16 holding 12-bit samples (J12SAMPLE rows)."""
        r = np.ascontiguousarray(rows, dtype=np.uint16 if np.asarray(rows).dtype == np.uint16 else np.uint8)
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
    w, h, nc, maxv, a = read_pnm(ppm)
    p = params_from_switches(switches, w, h, nc)
    img = pnm_samples(maxv, a, p.data_precision)[None]
    enc = encoder or Encoder(0)
    try:
        return enc.encode_batch(p, img)[0]
    finally:
        if encoder is None:
            enc.close()


def tj3_params(width: int, height: int, quality: int = 75, subsamp: str = "420", optimize: bool = False,
               progressive: bool = False, gray_input: bool = False, cmyk: bool = False, colorspace: int = None) -> Params:
    """The parameter block tj3Compress8 builds (turbojpeg.c:330-397
    setCompDefaults): JCP_FASTEST, quality via jpeg_set_quality(.., TRUE),
    YCbCr (or grayscale) with the luma sampling factors of TJSAMP_*.
    cmyk: TJPF_CMYK pixels, written as YCCK unless ``colorspace`` (TJPARAM_COLORSPACE as a CS_* value) says
    otherwise; component 3 gets the luma sampling factors."""
    p = Params()
    p.in_color_space = A.CS_GRAYSCALE if gray_input else (A.CS_CMYK if cmyk else A.CS_RGB)
    p.input_components = 1 if gray_input else (4 if cmyk else 3)
    p.data_precision = 8
    p.image_width, p.image_height = width, height
    _lib.b200jpeg_set_defaults(C.byref(p), A.PROFILE_FASTEST)
    p.image_width, p.image_height = width, height
    p.optimize_coding = int(optimize)
    _lib.b200jpeg_set_quality(C.byref(p), quality, 1)
    gray = gray_input or subsamp == "gray"
    if colorspace is None:
        colorspace = A.CS_GRAYSCALE if gray else (A.CS_YCCK if cmyk else A.CS_YCbCr)
    A.check(_lib.b200jpeg_set_colorspace(C.byref(p), colorspace), "set_colorspace")
    if progressive:
        A.check(_lib.b200jpeg_simple_progression(C.byref(p)), "simple_progression")
    hv = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2), "411": (4, 1), "441": (1, 4), "gray": (1, 1)}[subsamp]
    p.comp_info[0].h_samp_factor, p.comp_info[0].v_samp_factor = hv
    for ci in range(1, p.num_components):
        p.comp_info[ci].h_samp_factor = p.comp_info[ci].v_samp_factor = 1
    if p.num_components > 3:
        p.comp_info[3].h_samp_factor, p.comp_info[3].v_samp_factor = hv
    return p


def quality_tables(p: Params, qualities: Sequence[int], force_baseline: bool = True) -> np.ndarray:
    """Per-image quantization tables for Encoder.encode_batch(..., qtables=): (len(qualities), 4, 64) uint16, natural
    order.  Set i is what jpeg_set_quality(cinfo, qualities[i], force_baseline) leaves in quant_tbl when applied to a
    copy of ``p`` (jcparam.c:351-373: the scaled base tables of p.quant_tbl_master_idx in slots 0 and 1, the other
    slots as p has them).  It is jpeg_set_quality semantics only: unlike cjpeg's -quality switch it does not change
    the sampling factors at quality 80 and above."""
    out = np.zeros((len(qualities), A.NUM_QUANT_TBLS, 64), dtype=np.uint16)
    for i, q in enumerate(qualities):
        c = p.copy()
        _lib.b200jpeg_set_quality(C.byref(c), int(q), int(bool(force_baseline)))
        out[i] = np.ctypeslib.as_array(c.quant_tbl)
    return out
