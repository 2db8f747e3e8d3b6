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
from .cjpeg import decompress_options, params_for_jpeg_input, params_from_switches, pnm_samples, read_pnm, read_ppm  # noqa: F401

_lib = A.load()          # raises ImportError with build instructions if missing

__all__ = ["Encoder", "Params", "params_from_switches", "read_ppm", "cjpeg", "tj3_params", "quality_tables", "yuv_plane_dims", "B200JpegError"]


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

    # -- source files (device entropy decode of sequential Huffman JPEG files) ---------------------------------------
    @staticmethod
    def _files(files: Sequence[bytes]):
        bufs = [bytes(f) for f in files]
        ptrs = (C.c_void_p * len(bufs))(*[C.cast(C.c_char_p(b), C.c_void_p).value for b in bufs])
        sizes = (C.c_size_t * len(bufs))(*[len(b) for b in bufs])
        return bufs, ptrs, sizes

    def read_coefficients(self, files: Sequence[bytes]) -> List[np.ndarray]:
        """jpeg_read_coefficients for same-geometry files, decoded on the device: per component an (N, hib, wib, 64)
        int16 array of quantized coefficients in natural order (libjpeg JBLOCKs)."""
        info = _parse_first(files)
        bufs, ptrs, sizes = self._files(files)
        n = len(bufs)
        hmax = max(info.h_samp_factor[c] for c in range(info.num_components))
        vmax = max(info.v_samp_factor[c] for c in range(info.num_components))
        out = []
        for c in range(info.num_components):
            wib = -(-info.image_width * info.h_samp_factor[c] // (hmax * 8))
            hib = -(-info.image_height * info.v_samp_factor[c] // (vmax * 8))
            out.append(np.empty((n, hib, wib, 64), dtype=np.int16))
        k = len(out)
        A.check(_lib.b200jpeg_decode_coefs_batch(self._h, ptrs, sizes, n, (C.c_void_p * k)(*[a.ctypes.data for a in out]), 0,
                                                 (C.c_size_t * k)(*[a.shape[2] for a in out]),
                                                 (C.c_size_t * k)(*[a.shape[1] * a.shape[2] for a in out])), "decode_coefs_batch")
        return out

    def transcode_files(self, p: Params, files: Sequence[bytes]) -> List[bytes]:
        """b200jpeg_transcode_batch: the files decoded on the device and re-encoded with ``p`` (jpegtran.transcode
        builds it), each with the quantization tables its components latched."""
        bufs, ptrs, sizes = self._files(files)
        A.check(_lib.b200jpeg_transcode_batch(self._h, C.byref(p), ptrs, sizes, len(bufs)), "transcode_batch")
        return [self.get_output(i) for i in range(len(bufs))]

    def transcode_files_transform(self, p: Params, t: "A.TransformInfo", files: Sequence[bytes]) -> List[bytes]:
        """b200jpeg_transcode_batch_transform: transcode_files with the lossless transform ``t`` (b200jpeg_transform_setup
        filled it and ``p``) applied while the decoded coefficients are imported."""
        bufs, ptrs, sizes = self._files(files)
        A.check(_lib.b200jpeg_transcode_batch_transform(self._h, C.byref(p), C.byref(t), ptrs, sizes, len(bufs)), "transcode_batch_transform")
        return [self.get_output(i) for i in range(len(bufs))]

    def encode_batch_coefs_transform(self, p: Params, t: "A.TransformInfo", planes: Sequence[np.ndarray],
                                     qtables: Optional[np.ndarray] = None) -> List[bytes]:
        """b200jpeg_encode_batch_coefs_transform: planes[ci] is an (N, hib, wib, 64) int16 array in the SOURCE's
        geometry (any decoder's jpeg_read_coefficients output); qtables the sources' tables, (N, 4, 64) or None."""
        arrs = [np.ascontiguousarray(a, dtype=np.int16) for a in planes[:t.num_components]]
        n = arrs[0].shape[0]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        pitch = (C.c_size_t * len(arrs))(*[a.strides[1] // 128 for a in arrs])
        stride = (C.c_size_t * len(arrs))(*[a.strides[0] // 128 for a in arrs])
        q = None
        if qtables is not None:
            q, nq, _ = self._qtables(qtables, n)
            if nq != n:
                raise ValueError(f"qtables holds {nq} table sets for {n} images")
        A.check(_lib.b200jpeg_encode_batch_coefs_transform(self._h, C.byref(p), C.byref(t), ptrs, 0, pitch, stride,
                                                           None if q is None else q.ctypes.data_as(C.POINTER(C.c_uint16)), n),
                "encode_batch_coefs_transform")
        return [self.get_output(i) for i in range(n)]

    def decompress(self, files: Sequence[bytes], **opts) -> np.ndarray:
        """jpeg_read_scanlines for same-geometry sequential files, on the device: an (N, H, W, C) uint8 array, (N, H,
        W) for one output component.  Keyword options (decompress_options): scale=(num, denom), dct="int" | "fast" |
        "float", fancy=True, colorspace=None; without them a default decompress object (b200jpeg_decompress_batch)."""
        o = decompress_options(**opts) if opts else None
        w, h, _, nc = decompress_output(_parse_first(files), **opts)
        bufs, ptrs, sizes = self._files(files)
        out = np.empty((len(bufs), h, w, nc), dtype=np.uint8)
        if o is None:
            A.check(_lib.b200jpeg_decompress_batch(self._h, ptrs, sizes, len(bufs), out.ctypes.data, 0, out.strides[1], out.strides[0]), "decompress_batch")
        else:
            A.check(_lib.b200jpeg_decompress_batch_opts(self._h, C.byref(o), ptrs, sizes, len(bufs), out.ctypes.data, 0, out.strides[1], out.strides[0]),
                    "decompress_batch_opts")
        return out[..., 0] if nc == 1 else out

    def decompress_ptr(self, files: Sequence[bytes], ptr: int, row_pitch: int, image_stride: int, **opts) -> None:
        """Raw-pointer form of decompress: the pixels go to device memory at ``ptr`` and stay there."""
        bufs, ptrs, sizes = self._files(files)
        if not opts:
            A.check(_lib.b200jpeg_decompress_batch(self._h, ptrs, sizes, len(bufs), ptr, 1, row_pitch, image_stride), "decompress_batch")
        else:
            o = decompress_options(**opts)
            A.check(_lib.b200jpeg_decompress_batch_opts(self._h, C.byref(o), ptrs, sizes, len(bufs), ptr, 1, row_pitch, image_stride), "decompress_batch_opts")

    def recompress(self, p: Params, files: Sequence[bytes], **opts) -> List[bytes]:
        """cjpeg with JPEG input files (b200jpeg_recompress_batch): the files decoded to pixels on the device and
        encoded from there with ``p`` (cjpeg.params_for_jpeg_input builds it, with the same options); each output
        carries its source's COM and APPn segments as cjpeg copies them.  Keyword options as for decompress: a scaled
        rendition is recompressed from the scaled decode (b200jpeg_recompress_batch_opts)."""
        bufs, ptrs, sizes = self._files(files)
        if not opts:
            A.check(_lib.b200jpeg_recompress_batch(self._h, C.byref(p), ptrs, sizes, len(bufs)), "recompress_batch")
        else:
            o = decompress_options(**opts)
            A.check(_lib.b200jpeg_recompress_batch_opts(self._h, C.byref(o), C.byref(p), ptrs, sizes, len(bufs)), "recompress_batch_opts")
        return [self.get_output(i) for i in range(len(bufs))]

    def last_decode_sync(self):
        """(most rounds a CTA of the speculative decoder needed, subsequences the cross-CTA pass decoded again)."""
        r = C.c_int(0); q = C.c_longlong(0)
        A.check(_lib.b200jpeg_last_decode_sync(self._h, C.byref(r), C.byref(q)), "last_decode_sync")
        return r.value, q.value

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

    # -- YUV encoding (tj3EncodeYUVPlanes8) ---------------------------------
    def encode_yuv_batch(self, p: Params, images: np.ndarray) -> List[List[np.ndarray]]:
        """images: (N, H, W, C) or (N, H, W) uint8 host array -> per image, the list of its (ph, pw) uint8 planes
        (one per component of p, sizes from yuv_plane_dims), as tj3EncodeYUVPlanes8 writes them."""
        a = np.ascontiguousarray(images, dtype=np.uint8)
        if a.ndim == 3 and p.input_components == 1:
            a = a[..., None]
        n, h, w, c = a.shape
        if (w, h, c) != (p.image_width, p.image_height, p.input_components):
            raise ValueError("array shape does not match params")
        planes = [np.empty((n,) + yuv_plane_dims(p, ci)[::-1], dtype=np.uint8) for ci in range(p.num_components)]
        self.encode_yuv_batch_ptr(p, a.ctypes.data, False, a.strides[1], a.strides[0],
                                  [q.ctypes.data for q in planes], False, [q.strides[1] for q in planes], [q.strides[0] for q in planes], n)
        return [[q[i] for q in planes] for i in range(n)]

    def encode_yuv_batch_ptr(self, p: Params, ptr: int, on_device: bool, row_pitch: int, image_stride: int,
                             planes: Sequence[int], planes_on_device: bool, plane_pitch: Sequence[int], plane_stride: Sequence[int], n: int) -> None:
        """Raw-pointer form of encode_yuv_batch (device tensors, pinned host buffers): planes[ci] is image 0's plane of
        component ci, plane_pitch / plane_stride in bytes.  With pixels and planes on the device the call only enqueues."""
        k = len(planes)
        A.check(_lib.b200jpeg_encode_yuv_batch(self._h, C.byref(p), ptr, int(on_device), row_pitch, image_stride,
                                               (C.c_void_p * k)(*planes), int(planes_on_device), (C.c_size_t * k)(*plane_pitch),
                                               (C.c_size_t * k)(*plane_stride), n), "encode_yuv_batch")

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


def _parse_first(files: Sequence[bytes]) -> A.SourceInfo:
    if not len(files):
        raise ValueError("no files")
    info = A.SourceInfo()
    A.check(_lib.b200jpeg_parse_source(bytes(files[0]), len(files[0]), C.byref(info)), "parse_source: image 0")
    return info


def decompress_output(info: "A.SourceInfo", **opts):
    """(width, height, out_color_space, output_components) of a source decoded with the decompress defaults
    (b200jpeg_decompress_output): what rdjpeg.c copies into the compress object.  With keyword options
    (decompress_options) the same for a decompress object set up with them (b200jpeg_decompress_output_opts)."""
    w = C.c_int(0); h = C.c_int(0); cs = C.c_int(0); nc = C.c_int(0)
    if not opts:
        A.check(_lib.b200jpeg_decompress_output(C.byref(info), C.byref(w), C.byref(h), C.byref(cs), C.byref(nc)), "decompress_output")
    else:
        o = decompress_options(**opts)
        A.check(_lib.b200jpeg_decompress_output_opts(C.byref(info), C.byref(o), C.byref(w), C.byref(h), C.byref(cs), C.byref(nc)), "decompress_output_opts")
    return w.value, h.value, cs.value, nc.value


def cjpeg(switches: Sequence[str], ppm: bytes, encoder: Optional[Encoder] = None) -> bytes:
    """``cjpeg <switches> file`` on the device path: PPM/PGM or JPEG bytes -> JPEG bytes.  The input format follows
    cjpeg's select_file_type: a first byte 0xFF is a JPEG file, recompressed on the device."""
    if ppm[:1] == b"\xff":
        enc = encoder or Encoder(0)
        try:
            return enc.recompress(params_for_jpeg_input(switches, ppm), [ppm])[0]
        finally:
            if encoder is None:
                enc.close()
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
               progressive: bool = False, gray_input: bool = False, cmyk: bool = False, colorspace: int = None,
               pixel_format: str = None) -> Params:
    """The parameter block tj3Compress8 builds (turbojpeg.c:330-397
    setCompDefaults): JCP_FASTEST, quality via jpeg_set_quality(.., TRUE),
    YCbCr (or grayscale) with the luma sampling factors of TJSAMP_*.
    cmyk: TJPF_CMYK pixels, written as YCCK unless ``colorspace`` (TJPARAM_COLORSPACE as a CS_* value) says
    otherwise; component 3 gets the luma sampling factors.
    pixel_format: a TJPF_* name ("RGB", "BGR", "RGBX", ..., "ARGB", "GRAY", "CMYK") instead of gray_input / cmyk; the
    RGB family sets the matching JCS_EXT_* input order (pf2cs, turbojpeg.c)."""
    if pixel_format is not None:
        gray_input, cmyk = pixel_format == "GRAY", pixel_format == "CMYK"
    p = Params()
    p.in_color_space = A.CS_GRAYSCALE if gray_input else (A.CS_CMYK if cmyk else A.CS_RGB)
    p.input_components = 1 if gray_input else (4 if cmyk else 3)
    if pixel_format is not None and not (gray_input or cmyk):
        p.in_color_space, p.input_components = A.CS_EXT["EXT_" + pixel_format][:2]
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


def yuv_plane_dims(p: Params, ci: int):
    """(width, height) of plane ci of the YUV image Encoder.encode_yuv_batch writes (b200jpeg_yuv_plane_dims)."""
    w = C.c_int(0); h = C.c_int(0)
    A.check(_lib.b200jpeg_yuv_plane_dims(C.byref(p), ci, C.byref(w), C.byref(h)), "yuv_plane_dims")
    return w.value, h.value


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
