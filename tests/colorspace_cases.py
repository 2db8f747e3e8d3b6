"""Cases, images and reference access of the colour-space tests (tests/test_colorspaces.py) and of
tools/make_golden.py --colorspaces.  TEST INFRASTRUCTURE, not product code.

The reference side is build/librefcs.so (tests/refcs.c, compiled by __graft_entry__.build() where the reference
build under oracle/_ref/ exists): the unmodified reference library driven in cjpeg's call order, plus tj3Compress8."""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
from typing import Dict, List, Optional, Sequence

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "colorspace_golden.json")
REFCS = os.path.join(ROOT, "build", "librefcs.so")
REF = os.path.join(ROOT, "oracle", "_ref")

CS_UNKNOWN, CS_GRAYSCALE, CS_RGB, CS_YCbCr, CS_CMYK, CS_YCCK = 0, 1, 2, 3, 4, 5
CS_EXT_BGRX = 9

# name -> (in_color_space, input_components, jpeg_color_space or None for jpeg_default_colorspace)
CONVERSIONS = {
    "cmyk-cmyk": (CS_CMYK, 4, None),
    "cmyk-ycck": (CS_CMYK, 4, CS_YCCK),
    "ycck-ycck": (CS_YCCK, 4, None),
    "ycbcr-gray": (CS_YCbCr, 3, CS_GRAYSCALE),
    "unknown2": (CS_UNKNOWN, 2, None),
    "unknown4": (CS_UNKNOWN, 4, None),
}
# cjpeg's -revert re-runs jpeg_set_defaults, which re-applies jpeg_default_colorspace: under "cmyk-ycck" the -revert sets
# therefore encode CMYK->CMYK, as the reference's cjpeg does.  CMYK->YCCK under the fastest profile is covered by the
# TurboJPEG sets (tjopt: with optimal Huffman tables) and YCCK->YCCK by "ycck-ycck".
SWITCH_SETS = [
    ["-baseline", "-quality", "75"],
    ["-revert"],
    ["-revert", "-optimize"],
    ["-quality", "75"],
    ["-fastcrush", "-quality", "85"],
    ["-baseline", "-quality", "75", "-restart", "1"],
    ["-baseline", "-notrellis", "-quality", "60", "-sample", "2x2,1x1,1x1,2x2"],
    ["-baseline", "-quality", "75", "-smooth", "30"],
    ["-dct", "float"],
    ["-dct", "fast"],
    ["-precision", "12", "-notrellis", "-noovershoot", "-baseline"],
]
SIZES = [(1, 1), (17, 15), (227, 149)]
# TurboJPEG on TJPF_CMYK pixels: (name, TJSAMP_* value, optimize, progressive); TJSAMP_444 = 0, TJSAMP_420 = 2
TJ_SETS = [("tj420", 2, 0, 0), ("tj444", 0, 0, 0), ("tjprog", 2, 0, 1), ("tjopt", 2, 1, 0)]
TJ_COLORSPACES = {"cmyk-ycck": -1, "cmyk-cmyk": 3}     # -1: the library's choice (YCCK); 3 = TJCS_CMYK
TJ_SUBSAMP = {0: "444", 1: "422", 2: "420", 4: "440"}
RAW_CONVERSIONS = {"raw-cmyk": (CS_CMYK, CS_CMYK), "raw-ycck": (CS_YCCK, CS_YCCK)}
RAW_SETS = [["-baseline", "-quality", "75"], ["-revert"], ["-quality", "75"]]
TRAN_SOURCES = ["cmyk", "ycck"]                       # tj420 files of image seed 7, 227x149, written as CMYK / YCCK
TRAN_SETS = [[], ["-progressive"], ["-optimize"], ["-rotate", "90"], ["-crop", "96x64+16+8"]]


def precision_of(switches: Sequence[str]) -> int:
    return 12 if "-precision" in switches and switches[list(switches).index("-precision") + 1] == "12" else 8


def cmyk_image(seed: int, w: int, h: int, ncomp: int = 4, precision: int = 8) -> np.ndarray:
    """Seeded (h, w, ncomp) test image: smooth gradients, noise and, in every channel, runs of 0 and of MAXJSAMPLE
    (K-heavy areas, so that the deringing of blocks touching the maximum has work to do)."""
    maxj = 255 if precision == 8 else 4095
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.empty((h, w, ncomp), dtype=np.float64)
    for c in range(ncomp):
        fx, fy, ph = rng.uniform(0.01, 0.2), rng.uniform(0.01, 0.2), rng.uniform(0, 6.3)
        out[..., c] = (0.5 + 0.45 * np.sin(fx * x + fy * y + ph)) * maxj + rng.normal(0, maxj * 0.04, (h, w))
        for v in (0, maxj):                           # rectangles of 0 and MAXJSAMPLE, plus a full run in row 0
            x0, y0 = int(rng.integers(0, max(1, w))), int(rng.integers(0, max(1, h)))
            out[y0:y0 + max(1, h // 3), x0:x0 + max(1, w // 3), c] = v
        out[0, (c * 5) % w:(c * 5) % w + 4, c] = maxj
        if h > 1:
            out[h - 1, :max(1, w // 4), c] = 0
    return np.clip(np.rint(out), 0, maxj).astype(np.uint8 if precision == 8 else np.uint16)


def have_reference() -> bool:
    return os.path.exists(REFCS)


_lib = None


def refcs() -> C.CDLL:
    global _lib
    if _lib is None:
        lib = C.CDLL(REFCS)
        u8p = C.POINTER(C.c_ubyte)
        lib.refcs_encode.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.POINTER(C.c_char_p), C.POINTER(u8p), C.POINTER(C.c_ulong), C.c_char_p, C.c_int]
        lib.refcs_encode.restype = C.c_int
        lib.refcs_encode_tj_cmyk.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.POINTER(u8p), C.POINTER(C.c_ulong), C.c_char_p, C.c_int]
        lib.refcs_encode_tj_cmyk.restype = C.c_int
        lib.refcs_free.argtypes = [C.c_void_p]; lib.refcs_tjfree.argtypes = [C.c_void_p]
        _lib = lib
    return _lib


class RefError(RuntimeError):
    pass


def ref_encode(img: Optional[np.ndarray], in_cs: int, ic: int, jcs: Optional[int], switches: Sequence[str],
               planes: Optional[Sequence[np.ndarray]] = None, size=None) -> bytes:
    """The reference's file for pixels ``img`` (h, w, ic), or for raw-data ``planes`` with image size ``size``."""
    lib = refcs()
    argv = (C.c_char_p * max(1, len(switches)))(*[s.encode() for s in switches])
    out = C.POINTER(C.c_ubyte)(); n = C.c_ulong(0); err = C.create_string_buffer(256)
    if planes is not None:
        arrs = [np.ascontiguousarray(p, dtype=np.uint8) for p in planes]
        pp = (C.c_void_p * 4)(*[a.ctypes.data for a in arrs]); pitch = (C.c_int * 4)(*[a.strides[0] for a in arrs])
        w, h = size
        rc = lib.refcs_encode(None, 0, pp, pitch, w, h, in_cs, ic, -1 if jcs is None else jcs, len(switches), argv, C.byref(out), C.byref(n), err, 256)
    else:
        a = np.ascontiguousarray(img)
        h, w = a.shape[:2]
        rc = lib.refcs_encode(a.ctypes.data, w * ic, None, None, w, h, in_cs, ic, -1 if jcs is None else jcs, len(switches), argv, C.byref(out), C.byref(n), err, 256)
    if rc:
        raise RefError(err.value.decode())
    data = C.string_at(out, n.value)
    lib.refcs_free(out)
    return data


def ref_encode_tj(img: np.ndarray, quality: int, subsamp: int, optimize: int, progressive: int, colorspace: int) -> bytes:
    lib = refcs()
    a = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = a.shape[:2]
    out = C.POINTER(C.c_ubyte)(); n = C.c_ulong(0); err = C.create_string_buffer(256)
    if lib.refcs_encode_tj_cmyk(a.ctypes.data, w, h, quality, subsamp, optimize, progressive, colorspace, C.byref(out), C.byref(n), err, 256):
        raise RefError(err.value.decode())
    data = C.string_at(out, n.value)
    lib.refcs_tjfree(out)
    return data


def raw_planes(seed: int, p, ncomp: int) -> List[np.ndarray]:
    """Component planes of hib*8 x wib*8 samples for the geometry of params ``p`` (jcmaster.c:221-226)."""
    hmax = max(p.comp_info[ci].h_samp_factor for ci in range(ncomp)); vmax = max(p.comp_info[ci].v_samp_factor for ci in range(ncomp))
    out = []
    for ci in range(ncomp):
        h, v = p.comp_info[ci].h_samp_factor, p.comp_info[ci].v_samp_factor
        wib = -(-p.image_width * h // (hmax * 8)); hib = -(-p.image_height * v // (vmax * 8))
        out.append(cmyk_image(seed + 17 * ci, wib * 8, hib * 8, 1)[..., 0])
    return out


def md5(b: bytes) -> str:
    return hashlib.md5(b).hexdigest()


def case_id(*parts) -> str:
    return "|".join(str(x) for x in parts)


def pixel_cases() -> List[Dict]:
    """Every (conversion, switch set, size) and TurboJPEG case: id, inputs and how to build them."""
    cases = []
    for conv, (in_cs, ic, jcs) in CONVERSIONS.items():
        for sw in SWITCH_SETS:
            for (w, h) in SIZES:
                cases.append(dict(id=case_id(conv, " ".join(sw), f"{w}x{h}"), kind="cjpeg", conv=conv, switches=sw, w=w, h=h, seed=w * 7 + h))
    for conv in TJ_COLORSPACES:
        for name, ss, opt, prog in TJ_SETS:
            for (w, h) in SIZES:
                cases.append(dict(id=case_id(conv, name, f"{w}x{h}"), kind="tj", conv=conv, tj=[ss, opt, prog], w=w, h=h, seed=w * 7 + h))
    cases.append(dict(id=case_id("cmyk-ycck", "tj420", "1920x1080"), kind="tj", conv="cmyk-ycck", tj=[2, 0, 0], w=1920, h=1080, seed=3))
    return cases


def case_image(c: Dict) -> np.ndarray:
    in_cs, ic, _ = CONVERSIONS[c["conv"]]
    prec = precision_of(c.get("switches", []))
    return cmyk_image(c["seed"], c["w"], c["h"], ic, prec)


def reference_file(c: Dict) -> bytes:
    in_cs, ic, jcs = CONVERSIONS[c["conv"]]
    img = case_image(c)
    if c["kind"] == "tj":
        ss, opt, prog = c["tj"]
        return ref_encode_tj(img, 75, ss, opt, prog, TJ_COLORSPACES[c["conv"]])
    return ref_encode(img, in_cs, ic, jcs, c["switches"])


def tran_source(kind: str) -> bytes:
    """The jpegtran cases' source files: tj420 encodes of one CMYK image, as CMYK and as YCCK."""
    return ref_encode_tj(cmyk_image(7, 227, 149), 75, 2, 0, 0, 3 if kind == "cmyk" else -1)


def cmyk_to_ycck(img: np.ndarray, precision: int = 8) -> np.ndarray:
    """cmyk_ycck_convert (jccolor.c:395-441) restated: R, G, B = MAXJSAMPLE - C, M, Y (12-bit samples masked like
    RANGE_LIMIT) through the rgb_ycc_tab sums (jccolor.c:213-246: FIX(0.29900) = 19595, ...); K passes through as is."""
    maxj = 255 if precision == 8 else 4095
    centre = (maxj + 1) // 2
    a = img.astype(np.int64)
    r, g, b = (maxj - (a[..., k] & 0xFFF) for k in range(3))
    out = np.empty_like(img)
    out[..., 0] = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16
    out[..., 1] = (-11059 * r - 21709 * g + 32768 * b + (centre << 16) + 32767) >> 16
    out[..., 2] = (32768 * r - 27439 * g - 5329 * b + (centre << 16) + 32767) >> 16
    out[..., 3] = img[..., 3]
    return out


def _adobe_transform(jpeg: bytes, value: int) -> bytes:
    i = jpeg.find(b"\xff\xee\x00\x0eAdobe")
    assert i >= 0, "no Adobe APP14 segment"
    return jpeg[:i + 15] + bytes([value]) + jpeg[i + 16:]


def oracle_encode(p, img: np.ndarray, want_debug: bool = False):
    """The CPU restatement (oracle/jpeg_oracle.c) on a case of this file.  Its colour stage knows RGB->YCbCr / gray and
    null_convert, and its APP14 writer transform values 1 (YCbCr) and 0, so CMYK->YCCK runs as cmyk_to_ycck above followed
    by the restatement's null conversion of YCCK -- everything downstream of jccolor.c is the same in the reference --
    and YCCK files get the transform value 2 of jcmarker.c:596-606 here.  Returns oracle.OracleResult."""
    from oracle import oracle as O
    q = p.copy()
    if p.in_color_space == CS_CMYK and p.jpeg_color_space == CS_YCCK:
        q.in_color_space = CS_YCCK
        img = cmyk_to_ycck(img, p.data_precision)
    r = O.oracle_encode(q, img, want_debug)
    if p.jpeg_color_space == CS_YCCK and p.write_Adobe_marker:
        r.jpeg = _adobe_transform(r.jpeg, 2)
    return r


def oracle_encode_raw(p, planes) -> bytes:
    """The restatement on raw-data planes (already in the JPEG colour space), with YCCK's APP14 transform value."""
    from oracle import oracle as O
    out = O.oracle_encode_raw(p, planes)
    return _adobe_transform(out, 2) if p.jpeg_color_space == CS_YCCK and p.write_Adobe_marker else out


def load_golden() -> Dict:
    with open(GOLDEN) as f:
        return json.load(f)
