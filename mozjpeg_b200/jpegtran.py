"""Host-side mirror of the reference's ``jpegtran`` front end, encode half.

jpegtran (jpegtran.c:505-790) decodes a JPEG file to its quantized DCT
coefficients (jpeg_read_coefficients), copies the critical parameters into a
fresh compression object (jpeg_copy_critical_parameters, jctrans.c:76-166),
applies its switches and re-encodes with jpeg_write_coefficients - by default
with mozjpeg's scan search and optimal Huffman tables, which is the original
"jpegrescan" use of the library.  The decoder is out of this repo's scope:
the caller brings the coefficient planes (any JPEG decoder's
``jpeg_read_coefficients`` output); this file rebuilds the parameter block
from the source file's header and sequences the same API calls,

    jpeg_create_compress ; parse_switches(for_real=FALSE)        jpegtran.c:545-556
    jpeg_copy_critical_parameters                                jpegtran.c:700
    jtransform_adjust_parameters (1x1 sampling for gray sources) jpegtran.c:706
    parse_switches(for_real=TRUE)                                jpegtran.c:737
    jpeg_write_coefficients ; jpeg_finish_compress               jpegtran.c:750-765
    keep the input if it is smaller (prefer_smallest)            jpegtran.c:772-775

Lossless transforms (-rotate, -crop, ...), marker copying and arithmetic
coding are outside the hot path.  All parameter arithmetic happens in
libb200jpeg (params.cpp).
"""
from __future__ import annotations

import ctypes as C
import struct
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import _abi as A
from .cjpeg import UsageError, _keymatch

_ZZ = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
       35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]


class SourceInfo:
    """What jpeg_read_header leaves in a jpeg_decompress_struct, as far as jpeg_copy_critical_parameters reads it."""

    def __init__(self) -> None:
        self.image_width = self.image_height = 0
        self.data_precision = 8
        self.num_components = 0
        self.comps: List[Tuple[int, int, int, int]] = []        # (component_id, h, v, quant_tbl_no)
        self.quant: Dict[int, List[int]] = {}                    # slot -> 64 values, natural order
        self.saw_JFIF = False
        self.JFIF_version = (1, 1)
        self.density = (0, 1, 1)                                 # unit, X, Y
        self.saw_Adobe = False
        self.Adobe_transform = 0
        self.jpeg_color_space = A.CS_YCbCr
        self.has_extra_markers = False                           # COM / APPn other than JFIF and Adobe


def parse_header(jpeg: bytes) -> SourceInfo:
    """The marker segments up to the first SOS (jdmarker.c read_markers), then the colour-space guess of
    default_decompress_parms (jdapimin.c:111-213) for 1- and 3-component files."""
    s = SourceInfo()
    if jpeg[:2] != b"\xff\xd8":
        raise ValueError("not a JPEG file")
    pos = 2
    while pos + 4 <= len(jpeg):
        if jpeg[pos] != 0xFF:
            raise ValueError("corrupt JPEG header")
        m = jpeg[pos + 1]
        if m == 0xFF:
            pos += 1
            continue
        ln = struct.unpack(">H", jpeg[pos + 2:pos + 4])[0]
        seg = jpeg[pos + 4:pos + 2 + ln]
        if m in (0xC0, 0xC1, 0xC2):
            s.data_precision, s.image_height, s.image_width, nc = struct.unpack(">BHHB", seg[:6])
            s.num_components = nc
            for i in range(nc):
                cid, hv, tq = seg[6 + 3 * i:9 + 3 * i]
                s.comps.append((cid, hv >> 4, hv & 15, tq))
        elif m in (0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF):
            raise ValueError("lossless / hierarchical / arithmetic-coded source files are out of scope")
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                q += 1
                vals = [0] * 64
                for k in range(64):
                    if pq:
                        v = struct.unpack(">H", seg[q:q + 2])[0]; q += 2
                    else:
                        v = seg[q]; q += 1
                    vals[_ZZ[k]] = v
                s.quant[tq] = vals
        elif m == 0xE0 and seg[:5] == b"JFIF\0" and len(seg) >= 14:
            s.saw_JFIF = True
            s.JFIF_version = (seg[5], seg[6])
            s.density = (seg[7], struct.unpack(">H", seg[8:10])[0], struct.unpack(">H", seg[10:12])[0])
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            s.saw_Adobe = True
            s.Adobe_transform = seg[11]
        elif m == 0xFE or 0xE0 <= m <= 0xEF:
            s.has_extra_markers = True
        elif m == 0xDA:
            break
        pos += 2 + ln
    if s.num_components == 1:
        s.jpeg_color_space = A.CS_GRAYSCALE
    elif s.num_components == 3:
        ids = [c[0] for c in s.comps]
        if s.saw_JFIF:
            s.jpeg_color_space = A.CS_YCbCr
        elif s.saw_Adobe:
            s.jpeg_color_space = A.CS_RGB if s.Adobe_transform == 0 else A.CS_YCbCr
        elif ids == [1, 2, 3]:
            s.jpeg_color_space = A.CS_YCbCr
        elif ids == [0x52, 0x47, 0x42]:
            s.jpeg_color_space = A.CS_RGB
        else:
            s.jpeg_color_space = A.CS_YCbCr
    elif s.num_components == 4:
        # Adobe transform 2 marks YCCK, anything else (or no Adobe marker) CMYK
        s.jpeg_color_space = A.CS_YCCK if s.saw_Adobe and s.Adobe_transform == 2 else A.CS_CMYK
    else:
        raise ValueError("only 1-, 3- and 4-component files are on the device path")
    return s


class ConversionError(ValueError):
    """The reference refuses the request with JERR_CONVERSION_NOTIMPL and writes no file."""


def _copy_critical_parameters(src: SourceInfo, profile: int) -> A.Params:
    """jpeg_copy_critical_parameters (jctrans.c:76-166) on an object whose compression profile is ``profile``."""
    lib = A.load()
    p = A.Params()
    p.image_width, p.image_height = src.image_width, src.image_height
    p.input_components = src.num_components
    p.in_color_space = src.jpeg_color_space
    p.data_precision = 8
    lib.b200jpeg_set_defaults(C.byref(p), profile)                       # jctrans.c:102
    p.trellis_quant = 0                                                  # jctrans.c:103
    A.check(lib.b200jpeg_set_colorspace(C.byref(p), src.jpeg_color_space), "set_colorspace")
    p.data_precision = src.data_precision
    for slot, vals in src.quant.items():
        for k in range(64):
            p.quant_tbl[slot][k] = vals[k]
        p.quant_tbl_present[slot] = 1
    p.num_components = src.num_components
    for ci, (cid, h, v, tq) in enumerate(src.comps):
        c = p.comp_info[ci]
        c.component_id, c.h_samp_factor, c.v_samp_factor, c.quant_tbl_no = cid, h, v, tq
        if tq not in src.quant:
            raise ValueError(f"Quantization table 0x{tq:02x} was not defined")
    if src.saw_JFIF:
        if src.JFIF_version[0] == 1:
            p.JFIF_major_version, p.JFIF_minor_version = src.JFIF_version
        p.density_unit, p.X_density, p.Y_density = src.density
    return p


def _parse(p: A.Params, argv: Sequence[str], for_real: bool) -> bool:
    """parse_switches (jpegtran.c:133-466), the switches that reach the encoder.  Returns prefer_smallest."""
    lib = A.load()
    simple_progressive = p.num_scans != 0            # jpegtran.c:154
    prefer_smallest = True
    i, n = 0, len(argv)
    while i < n:
        arg = argv[i]
        if not arg.startswith("-"):
            raise UsageError(f"unexpected file argument {arg!r}")
        a = arg[1:]
        if _keymatch(a, "copy", 2):
            i += 1
            if i >= n or not (_keymatch(argv[i], "none", 1)):
                raise UsageError("only -copy none is on the device path (no marker copying)")
        elif _keymatch(a, "fastcrush", 4):
            p.optimize_scans = 0
        elif _keymatch(a, "optimize", 1) or _keymatch(a, "optimise", 1):
            p.optimize_coding = 1
        elif _keymatch(a, "progressive", 1):
            simple_progressive = True
            prefer_smallest = False
        elif _keymatch(a, "restart", 1):
            i += 1
            if i >= n:
                raise UsageError("missing argument for restart")
            v = argv[i]
            if v[-1:] in "bB":
                p.restart_interval = int(v[:-1]); p.restart_in_rows = 0
            else:
                p.restart_in_rows = int(v)
        elif _keymatch(a, "revert", 3):
            p.compress_profile = A.PROFILE_FASTEST        # only the profile: no jpeg_set_defaults here (jpegtran.c:378-381)
            prefer_smallest = False
        else:
            raise UsageError(f"unknown or out-of-scope option {arg!r}")
        i += 1
    if for_real and simple_progressive:
        A.check(lib.b200jpeg_simple_progression(C.byref(p)), "simple_progression")
    return prefer_smallest


def params_for_transcode(src: SourceInfo, switches: Sequence[str]) -> Tuple[A.Params, bool]:
    """(dstinfo at jpeg_write_coefficients, prefer_smallest) for ``jpegtran <switches> file``."""
    # first pass on the bare object (profile JCP_MAX_COMPRESSION, jcapimin.c:108): everything it sets is overwritten by
    # the jpeg_set_defaults inside jpeg_copy_critical_parameters - except the profile itself, which that call reads
    if any(_keymatch(a[1:], "grayscale", 2) or _keymatch(a[1:], "greyscale", 2) for a in switches if a.startswith("-")):
        if src.num_components == 4:                   # jtransform_adjust_parameters (transupp.c:2048-2071)
            raise ConversionError("Unsupported color conversion request")
        raise UsageError("-grayscale is not on the device path")
    p0 = A.Params()
    p0.compress_profile = A.PROFILE_MAX_COMPRESSION
    _parse(p0, list(switches), False)
    p = _copy_critical_parameters(src, p0.compress_profile)
    if src.num_components == 1:                       # jtransform_adjust_parameters (transupp.c:2072-2079): a single-component
        p.comp_info[0].h_samp_factor = 1              # source always leaves with 1x1 sampling, with or without -grayscale
        p.comp_info[0].v_samp_factor = 1
    prefer_smallest = _parse(p, list(switches), True)
    if p.num_scans == 0:                              # jpeg_write_coefficients has no such step; kept for symmetry with
        p.optimize_scans = 0                          # jpeg_start_compress (a sequential file has nothing to search)
    return p, prefer_smallest


def _same_except_quant(a: SourceInfo, b: SourceInfo) -> bool:
    """Everything jpeg_copy_critical_parameters reads from a source, except the quantization tables' values: geometry,
    components, sampling, slot mapping and defined slots, precision, colour space, JFIF fields."""
    keys = ("image_width", "image_height", "data_precision", "num_components", "comps", "jpeg_color_space",
            "saw_JFIF", "JFIF_version", "density", "saw_Adobe", "Adobe_transform")
    return all(getattr(a, k) == getattr(b, k) for k in keys) and sorted(a.quant) == sorted(b.quant)


def transcode(encoder, sources: Sequence[bytes], coef_planes: Sequence[Sequence], switches: Sequence[str]) -> List[bytes]:
    """``jpegtran <switches>`` on same-shaped source files: sources[i] is the original file, coef_planes[ci] an
    (N, height_in_blocks, width_in_blocks, 64) int16 array of its quantized coefficients (natural order).
    Every source keeps its own quantization tables (its DQT); everything else jpeg_copy_critical_parameters takes
    from a source must match the first one, else ValueError names the first source that differs."""
    infos = [parse_header(s) for s in sources]
    for i, info in enumerate(infos[1:], 1):
        if not _same_except_quant(infos[0], info):
            raise ValueError(f"source {i} differs from source 0 in more than its quantization tables")
    p, prefer_smallest = params_for_transcode(infos[0], switches)
    qt = np.zeros((len(infos), A.NUM_QUANT_TBLS, 64), dtype=np.uint16)
    for i, info in enumerate(infos):
        qt[i] = np.ctypeslib.as_array(p.quant_tbl)
        for slot, vals in info.quant.items():
            qt[i, slot] = vals
    out = encoder.encode_batch_coefs(p, coef_planes, qtables=qt)
    if prefer_smallest and p.compress_profile == A.PROFILE_MAX_COMPRESSION:
        out = [s if len(s) < len(o) else o for s, o in zip(sources, out)]      # jpegtran.c:772-775
    return out
