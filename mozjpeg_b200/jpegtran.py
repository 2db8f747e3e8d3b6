"""Host-side mirror of the reference's ``jpegtran`` front end, encode half.

jpegtran (jpegtran.c:505-790) decodes a JPEG file to its quantized DCT
coefficients (jpeg_read_coefficients), copies the critical parameters into a
fresh compression object (jpeg_copy_critical_parameters, jctrans.c:76-166),
applies its switches and re-encodes with jpeg_write_coefficients - by default
with mozjpeg's scan search and optimal Huffman tables, which is the original
"jpegrescan" use of the library.  The coefficient planes come from the
library's device entropy decode of sequential Huffman files, or from the
caller (any JPEG decoder's ``jpeg_read_coefficients`` output, e.g. for
progressive sources); this file rebuilds the parameter block from the source
file's header and sequences the same API calls,

    jpeg_create_compress ; parse_switches(for_real=FALSE)        jpegtran.c:545-556
    jpeg_copy_critical_parameters                                jpegtran.c:700
    jtransform_adjust_parameters (1x1 sampling for gray sources) jpegtran.c:706
    parse_switches(for_real=TRUE)                                jpegtran.c:737
    jpeg_write_coefficients ; jpeg_finish_compress               jpegtran.c:750-765
    keep the input if it is smaller (prefer_smallest)            jpegtran.c:772-775

The lossless transforms (-rotate, -flip, -transpose, -transverse, -crop, -trim,
-perfect, -grayscale) run on the device too: b200jpeg_transform_setup
(transform.cpp, jtransform_request_workspace + jtransform_adjust_parameters)
sits between jpeg_copy_critical_parameters and the for-real switch pass, and
the coefficient import applies the block mapping of transupp.c's do_* routines.
-drop, -wipe, crop extension, marker copying and arithmetic coding stay the
reference's.  All parameter arithmetic happens in libb200jpeg (params.cpp,
transform.cpp).
"""
from __future__ import annotations

import ctypes as C
import struct
from typing import Dict, List, Optional, Sequence, Tuple

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


def parse_source(jpeg: bytes) -> A.SourceInfo:
    """b200jpeg_parse_source: every marker segment and scan of the file (ValueError with the library's message when it
    refuses the file)."""
    out = A.SourceInfo()
    rc = A.load().b200jpeg_parse_source(bytes(jpeg), len(jpeg), C.byref(out))
    if rc < 0:
        raise ValueError(A.load().b200jpeg_last_error().decode("utf-8", "replace"))
    return out


def parse_header(jpeg: bytes) -> SourceInfo:
    """The marker segments up to the first SOS (jdmarker.c read_markers), then the colour-space guess of
    default_decompress_parms (jdapimin.c:111-213) for 1- and 3-component files; parsed by b200jpeg_parse_source."""
    r = parse_source(jpeg)
    s = SourceInfo()
    s.image_width, s.image_height, s.data_precision, s.num_components = r.image_width, r.image_height, r.data_precision, r.num_components
    s.comps = [(r.component_id[i], r.h_samp_factor[i], r.v_samp_factor[i], r.quant_tbl_no[i]) for i in range(r.num_components)]
    s.quant = {t: list(r.quant_tbl[t]) for t in range(A.NUM_QUANT_TBLS) if r.quant_tbl_present[t]}
    s.saw_JFIF = bool(r.saw_JFIF)
    s.JFIF_version = (r.JFIF_major_version, r.JFIF_minor_version)
    s.density = (r.density_unit, r.X_density, r.Y_density)
    s.saw_Adobe = bool(r.saw_Adobe)
    s.Adobe_transform = r.Adobe_transform
    s.jpeg_color_space = r.jpeg_color_space
    s.has_extra_markers = bool(r.has_extra_markers)
    return s


class ConversionError(ValueError):
    """The reference refuses the request with JERR_CONVERSION_NOTIMPL and writes no file."""


class TransformError(ValueError):
    """The reference refuses the transform request and writes no file: "transformation is not perfect" (-perfect) or
    "Invalid crop request" (JERR_BAD_CROP_SPEC)."""


def _read_uint(spec: str, i: int) -> Tuple[Optional[int], int]:
    """jt_read_integer (transupp.c:1365-1379): decimal digits as a JDIMENSION (wrapping like the unsigned arithmetic)."""
    j, v = i, 0
    while j < len(spec) and spec[j] in "0123456789":
        v = (v * 10 + ord(spec[j]) - 48) & 0xFFFFFFFF
        j += 1
    return (v, j) if j > i else (None, i)


def parse_crop_spec(t: A.TransformInfo, spec: str) -> bool:
    """jtransform_parse_crop_spec (transupp.c:1395-1450): <width>[{fr}]x<height>[{fr}]{+-}<xoffset>{+-}<yoffset>."""
    t.crop = 0
    t.crop_width_set = t.crop_height_set = t.crop_xoffset_set = t.crop_yoffset_set = A.CROP_UNSET
    i = 0
    kinds = {"f": A.CROP_FORCE, "r": A.CROP_REFLECT}
    if spec[i:i + 1] in tuple("0123456789"):
        t.crop_width, i = _read_uint(spec, i)
        t.crop_width_set = kinds.get(spec[i:i + 1].lower(), A.CROP_POS)
        i += t.crop_width_set != A.CROP_POS
    if spec[i:i + 1] in ("x", "X"):
        v, i = _read_uint(spec, i + 1)
        if v is None:
            return False
        t.crop_height = v
        t.crop_height_set = kinds.get(spec[i:i + 1].lower(), A.CROP_POS)
        i += t.crop_height_set != A.CROP_POS
    for off in ("crop_xoffset", "crop_yoffset"):
        if spec[i:i + 1] in ("+", "-"):
            setattr(t, off + "_set", A.CROP_NEG if spec[i] == "-" else A.CROP_POS)
            v, i = _read_uint(spec, i + 1)
            if v is None:
                return False
            setattr(t, off, v)
    if i != len(spec):
        return False
    t.crop = 1
    return True


def _source_struct(src: SourceInfo) -> A.SourceInfo:
    """The fields of b200jpeg_source_info that b200jpeg_transform_setup reads."""
    r = A.SourceInfo()
    r.image_width, r.image_height, r.data_precision, r.num_components = src.image_width, src.image_height, src.data_precision, src.num_components
    for ci, (cid, h, v, tq) in enumerate(src.comps):
        r.component_id[ci], r.h_samp_factor[ci], r.v_samp_factor[ci], r.quant_tbl_no[ci] = cid, h, v, tq
    r.jpeg_color_space = src.jpeg_color_space
    return r


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


def _parse(p: A.Params, argv: Sequence[str], for_real: bool, t: Optional[A.TransformInfo] = None) -> bool:
    """parse_switches (jpegtran.c:133-466), the switches that reach the encoder and, into ``t``, the transform
    switches.  Returns prefer_smallest."""
    lib = A.load()
    t = A.TransformInfo() if t is None else t
    C.memset(C.byref(t), 0, C.sizeof(t))                 # jpegtran.c:164-169
    simple_progressive = p.num_scans != 0            # jpegtran.c:154
    prefer_smallest = True
    i, n = 0, len(argv)

    def value(name: str) -> str:
        if i + 1 >= n:
            raise UsageError(f"missing argument for -{name}")
        return argv[i + 1]

    def select(x: int) -> None:                      # select_transform (jpegtran.c:112-130)
        if t.transform not in (A.XFORM_NONE, x):
            raise UsageError("can only do one image transformation at a time")
        t.transform = x

    while i < n:
        arg = argv[i]
        if not arg.startswith("-"):
            raise UsageError(f"unexpected file argument {arg!r}")
        a = arg[1:]
        if _keymatch(a, "copy", 2):
            i += 1
            if i >= n or not (_keymatch(argv[i], "none", 1)):
                raise UsageError("only -copy none is on the device path (no marker copying)")
        elif _keymatch(a, "crop", 2):
            spec = value("crop"); i += 1
            if t.crop or not parse_crop_spec(t, spec):
                raise UsageError(f"bogus -crop argument '{spec}'")
            prefer_smallest = False
        elif _keymatch(a, "drop", 2):
            raise UsageError("-drop is not on the device path")
        elif _keymatch(a, "flip", 1):
            v = value("flip"); i += 1
            if _keymatch(v, "horizontal", 1):
                select(A.XFORM_FLIP_H)
            elif _keymatch(v, "vertical", 1):
                select(A.XFORM_FLIP_V)
            else:
                raise UsageError(f"bad -flip argument {v!r}")
            prefer_smallest = False
        elif _keymatch(a, "fastcrush", 4):
            p.optimize_scans = 0
        elif _keymatch(a, "grayscale", 1) or _keymatch(a, "greyscale", 1):
            t.force_grayscale = 1
            prefer_smallest = False
        elif _keymatch(a, "optimize", 1) or _keymatch(a, "optimise", 1):
            p.optimize_coding = 1
        elif _keymatch(a, "perfect", 2):
            t.perfect = 1
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
        elif _keymatch(a, "rotate", 2):
            v = value("rotate"); i += 1
            angle = next((x for key, mn, x in (("90", 2, A.XFORM_ROT_90), ("180", 3, A.XFORM_ROT_180), ("270", 3, A.XFORM_ROT_270))
                          if _keymatch(v, key, mn)), None)
            if angle is None:
                raise UsageError(f"bad -rotate argument {v!r}")
            select(angle)
            prefer_smallest = False
        elif _keymatch(a, "transpose", 1):
            select(A.XFORM_TRANSPOSE)
            prefer_smallest = False
        elif _keymatch(a, "transverse", 6):
            select(A.XFORM_TRANSVERSE)
            prefer_smallest = False
        elif _keymatch(a, "trim", 3):
            t.trim = 1
            prefer_smallest = False
        elif _keymatch(a, "wipe", 1):
            raise UsageError("-wipe is not on the device path")
        else:
            raise UsageError(f"unknown or out-of-scope option {arg!r}")
        i += 1
    if for_real and simple_progressive:
        A.check(lib.b200jpeg_simple_progression(C.byref(p)), "simple_progression")
    return prefer_smallest


def transcode_setup(src: SourceInfo, switches: Sequence[str]) -> Tuple[A.Params, A.TransformInfo, bool]:
    """(dstinfo at jpeg_write_coefficients, the transform, prefer_smallest) for ``jpegtran <switches> file``."""
    # first pass on the bare object (profile JCP_MAX_COMPRESSION, jcapimin.c:108): everything it sets is overwritten by
    # the jpeg_set_defaults inside jpeg_copy_critical_parameters - except the profile itself, which that call reads
    p0 = A.Params()
    p0.compress_profile = A.PROFILE_MAX_COMPRESSION
    t = A.TransformInfo()
    _parse(p0, list(switches), False, t)
    p = _copy_critical_parameters(src, p0.compress_profile)
    # jtransform_request_workspace + jtransform_adjust_parameters (jpegtran.c:700-706): the destination's size, sampling,
    # tables and, under -grayscale, colour space, before the for-real pass builds e.g. the -progressive script for it
    rc = A.load().b200jpeg_transform_setup(C.byref(_source_struct(src)), C.byref(t), C.byref(p))
    if rc < 0:
        msg = A.load().b200jpeg_last_error().decode("utf-8", "replace")
        if "Unsupported color conversion" in msg:
            raise ConversionError(msg)
        if rc == A.ERR_UNSUPPORTED and "crop extension" in msg:
            raise UsageError(f"-crop: {msg}")
        if rc == A.ERR_PARAM and msg in ("transformation is not perfect", "Invalid crop request"):
            raise TransformError(msg)
        A.check(rc, "transform_setup")
    prefer_smallest = _parse(p, list(switches), True)
    if p.num_scans == 0:                              # jpeg_write_coefficients has no such step; kept for symmetry with
        p.optimize_scans = 0                          # jpeg_start_compress (a sequential file has nothing to search)
    return p, t, prefer_smallest


def params_for_transcode(src: SourceInfo, switches: Sequence[str]) -> Tuple[A.Params, bool]:
    """(dstinfo at jpeg_write_coefficients, prefer_smallest) for ``jpegtran <switches> file``."""
    p, _, prefer_smallest = transcode_setup(src, switches)
    return p, prefer_smallest


def _is_identity(t: A.TransformInfo) -> bool:
    return t.transform == A.XFORM_NONE and not t.crop and not t.force_grayscale


def _same_except_quant(a: SourceInfo, b: SourceInfo) -> bool:
    """Everything jpeg_copy_critical_parameters reads from a source, except the quantization tables' values: geometry,
    components, sampling, slot mapping and defined slots, precision, colour space, JFIF fields."""
    keys = ("image_width", "image_height", "data_precision", "num_components", "comps", "jpeg_color_space",
            "saw_JFIF", "JFIF_version", "density", "saw_Adobe", "Adobe_transform")
    return all(getattr(a, k) == getattr(b, k) for k in keys) and sorted(a.quant) == sorted(b.quant)


def transcode(encoder, sources: Sequence[bytes], coef_planes: Optional[Sequence[Sequence]], switches: Sequence[str]) -> List[bytes]:
    """``jpegtran <switches>`` on same-shaped source files: sources[i] is the original file, coef_planes[ci] an
    (N, height_in_blocks, width_in_blocks, 64) int16 array of its quantized coefficients (natural order), or None:
    the sources' entropy-coded data is then decoded on the device (sequential Huffman files, and progressive ones
    when the encoder's progressive decode is on; otherwise a progressive source raises ValueError, pass its planes
    instead).
    Every source keeps its own quantization tables (its DQT); everything else jpeg_copy_critical_parameters takes
    from a source must match the first one, else ValueError names the first source that differs."""
    infos = [parse_header(s) for s in sources]
    for i, info in enumerate(infos[1:], 1):
        if not _same_except_quant(infos[0], info):
            raise ValueError(f"source {i} differs from source 0 in more than its quantization tables")
    p, t, prefer_smallest = transcode_setup(infos[0], switches)
    identity = _is_identity(t)
    if coef_planes is None:
        try:
            out = encoder.transcode_files(p, sources) if identity else encoder.transcode_files_transform(p, t, sources)
        except A.B200JpegError as e:
            if e.code == A.ERR_UNSUPPORTED and "progressive" in str(e):
                raise ValueError(f"{e}: decode such sources with any JPEG decoder's jpeg_read_coefficients and pass "
                                 "their planes as coef_planes") from e
            raise
    else:
        qt = np.zeros((len(infos), A.NUM_QUANT_TBLS, 64), dtype=np.uint16)
        base = np.ctypeslib.as_array(p.quant_tbl).copy()
        if t.transposed:                              # the transform entry point takes the sources' orientation
            base = base.reshape(-1, 8, 8).transpose(0, 2, 1).reshape(-1, 64)
        for i, info in enumerate(infos):
            qt[i] = base
            for slot, vals in info.quant.items():
                qt[i, slot] = vals
        if identity:
            out = encoder.encode_batch_coefs(p, coef_planes, qtables=qt)
        else:
            out = encoder.encode_batch_coefs_transform(p, t, coef_planes, qtables=qt)
    if prefer_smallest and p.compress_profile == A.PROFILE_MAX_COMPRESSION:
        out = [s if len(s) < len(o) else o for s, o in zip(sources, out)]      # jpegtran.c:772-775
    return out


def main(argv: Sequence[str] = None) -> int:
    """``python -m mozjpeg_b200.jpegtran [switches] [-outfile name] file.jpg`` - jpegtran's command line on the device
    path, from the file's bytes (sequential and progressive Huffman sources, as the reference's jpegtran reads both)."""
    import sys
    from . import Encoder
    args = list(sys.argv[1:] if argv is None else argv)
    outfile = None
    switches: List[str] = []
    files: List[str] = []
    i = 0
    while i < len(args):
        a = args[i]
        if a.startswith("-") and len(a) > 1:
            if _keymatch(a[1:], "outfile", 4):
                if i + 1 >= len(args):
                    raise UsageError("missing argument for -outfile")
                outfile = args[i + 1]; i += 2; continue
            switches.append(a)
            takes_value = ("restart", 1), ("copy", 2), ("crop", 2), ("flip", 1), ("rotate", 2)
            if any(_keymatch(a[1:], k, m) for k, m in takes_value) and i + 1 < len(args):
                switches.append(args[i + 1]); i += 1
        else:
            files.append(a)
        i += 1
    if len(files) != 1:
        print("usage: python -m mozjpeg_b200.jpegtran [switches] [-outfile name] file.jpg", file=sys.stderr)
        return 2
    with open(files[0], "rb") as f:
        src = f.read()
    try:
        transcode_setup(parse_header(src), switches)
    except TransformError as e:
        if str(e) != "transformation is not perfect":
            raise
        print(f"jpegtran: {e}", file=sys.stderr)          # jpegtran.c:679-682
        return 1
    enc = Encoder(0)
    enc.set_progressive_decode(True)
    try:
        out = transcode(enc, [src], None, switches)[0]
    finally:
        enc.close()
    if outfile:
        with open(outfile, "wb") as fo:
            fo.write(out)
    else:
        sys.stdout.buffer.write(out)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
