"""Sources, options and expected results of the decompress-to-YUV tests (tests/test_yuv_decode.py) and of
tools/make_golden.py --yuv-decode.

Every source is written by the repository's CPU oracle (tests/decode_cases.py, tests/recompress_cases.py,
tests/progressive_cases.py), so a GPU run needs no stored JPEG file.  tests/golden/yuv_decode_golden.json records per
(source, scale, dct) what the reference's tj3DecompressToYUVPlanes8 (oracle/_ref/libturbojpeg_ref.so through ctypes)
reports: the TJSAMP_* of the source, each plane's pw x ph and the md5 of its defined samples, or its refusal.

The defined samples of plane ci are its first min(ih, ph) rows of min(iw, pw) samples, iw = width_in_blocks * k and
ih = height_in_blocks * k (k = 8 * num / denom): beyond them the reference copies bytes of its temporary buffer whose
contents depend on its heap layout, and the device writes nothing.  plan() restates getSubsamp, tj3YUVPlaneWidth /
Height and those sizes for the CPU tests.

The golden also records, for the sources of RECOMPRESS, the md5 of the reference's tj3DecompressToYUVPlanes8 followed by
tj3CompressFromYUVPlanes8 (quality 75, the source's subsampling), and for the decode direction (tj3DecodeYUVPlanes8)
the md5 of the pixels the reference makes from seeded planes (decode_planes) for every subsampling x pixel format but
CMYK x odd and even size x plane pitch, and its refusal of CMYK."""
import ctypes as C
import hashlib
import json
import os

import numpy as np

import decode_cases as D
import progressive_cases as P
import recompress_cases as R

ROOT = R.ROOT
GOLDEN = os.path.join(ROOT, "tests", "golden", "yuv_decode_golden.json")
REF_TJ = os.path.join(ROOT, "oracle", "_ref", "libturbojpeg_ref.so")

SUBSAMPS = ("444", "422", "420", "gray", "440", "411", "441")          # TJSAMP_* in enum order
MCU = {0: (8, 8), 1: (16, 8), 2: (16, 16), 3: (8, 8), 4: (8, 16), 5: (32, 8), 6: (8, 32)}
SCALES = [(1, 8), (1, 4), (1, 2), (1, 1)]
DCTS = ("int", "fast")

# decode_cases tuple format: (id, width, height, seed, cjpeg switches, layout)
LAYOUTS = [
    ("y_gray", 227, 149, 71, ["-revert", "-grayscale"], None),
    ("y_444", 227, 149, 72, ["-revert", "-sample", "1x1"], None),
    ("y_422", 227, 149, 73, ["-revert", "-sample", "2x1"], None),
    ("y_420", 227, 149, 74, ["-revert", "-sample", "2x2"], None),
    ("y_440", 227, 149, 75, ["-revert", "-sample", "1x2"], None),
    ("y_411", 227, 149, 76, ["-revert", "-sample", "4x1"], None),
    ("y_441", 227, 149, 77, ["-revert", "-sample", "1x4"], None),
    ("y_ns422", 227, 149, 78, ["-revert", "-sample", "2x2,1x2,1x2"], None),      # getSubsamp's non-standard 4:2:2
    ("y_ns440", 227, 149, 79, ["-revert", "-sample", "2x2,2x1,2x1"], None),      # and 4:4:0
    ("y_ns444", 227, 149, 80, ["-revert", "-sample", "1x2,1x2,1x2"], None),      # 4:4:4 at equal factors
    ("y_2x2x3", 227, 149, 81, ["-revert", "-sample", "2x2,2x2,2x2"], "multi"),   # equal 2x2 factors: one scan per component
    ("y_rgb", 227, 149, 82, ["-revert", "-rgb"], None),
]
SMALL = [
    ("y_1x1", 1, 1, 83, ["-revert", "-sample", "2x2"], None),
    ("y_2x3", 2, 3, 84, ["-revert", "-sample", "2x2"], None),
    ("y_3x1", 3, 1, 85, ["-revert", "-sample", "2x2"], None),
    ("y_1x3_411", 1, 3, 86, ["-revert", "-sample", "4x1"], None),
    ("y_3x2_441", 3, 2, 87, ["-revert", "-sample", "1x4"], None),
    ("y_3x3_422", 3, 3, 88, ["-revert", "-sample", "2x1"], None),
]
FOURK = ("y_4k", 3840, 2160, 89, ["-revert", "-quality", "90", "-sample", "2x2"], None)
_OWN = {c[0]: c for c in LAYOUTS + SMALL + [FOURK]}
# sources of recompress_cases (4:2:0, 200x136 and 203x131): quality extremes, a 16-bit DQT, restarts, one scan per component
CONTENT = ["q5", "q100", "sof1_dqt16", "restart_1", "restart_3B", "multi_scan"]
# progressive sources (progressive decode on)
PROGRESSIVE = ["prog:progressive", "prog:sample_420", "prog:sample_422"]
# refused by the device: 4 components, 3x2 sampling, 12 bits (the reference refuses these too), an incomplete progression
# the reference would block-smooth, and corrupt data
REFUSED_SOURCES = ["prog:cmyk", "prog:sample_3x2", "prog:prog12", "prog:drop_to_dc_only", "prog:corrupt"]
REFUSED_SCALES = [(3, 8), (3, 4)]


def source(sid):
    """file bytes of source ``sid``"""
    if sid.startswith("prog:"):
        name = sid[5:]
        if name in P.EXTRA_IDS:
            return P.extra_source(name)
        return P.source(next(c for c in P.CASES if c[0] == name))
    if sid in _OWN:
        if sid not in R._cache:
            R._cache[sid] = D.source(_OWN[sid])
        return R._cache[sid][0]
    return R.source(sid)[0]


def case_id(sid, scale, dct):
    return f"{sid}:{scale[0]}/{scale[1]}:{dct}"


def cases():
    """[(id, source id, (num, denom), dct)]"""
    out = []
    for lay in LAYOUTS:
        for sc in SCALES:
            for dct in DCTS:
                out.append((lay[0], sc, dct))
    for lay in SMALL:
        for sc in SCALES:
            out.append((lay[0], sc, "int"))
    for sid in CONTENT:
        for sc in SCALES:
            for dct in DCTS:
                out.append((sid, sc, dct))
    for sid in PROGRESSIVE:
        for sc in ((1, 1), (1, 2)):
            out.append((sid, sc, "fast" if sc == (1, 2) else "int"))
    out += [(FOURK[0], (1, 1), "int"), (FOURK[0], (1, 2), "fast"), (FOURK[0], (1, 4), "int")]
    for sid in REFUSED_SOURCES:
        out.append((sid, (1, 1), "int"))
    for sc in REFUSED_SCALES:
        out.append(("y_420", sc, "int"))
    return [(case_id(*c), *c) for c in out]


# decompress_yuv -> encode_batch_raw(tj3_params(.., quality 75, subsampling)): sources and options whose planes are
# fully defined (iw >= pw and ih >= ph for every plane)
RECOMPRESS = [("y_420", (1, 1), "int"), ("y_420", (1, 2), "fast"), ("y_422", (1, 1), "int"), ("y_gray", (1, 1), "int"),
              ("y_444", (1, 4), "int"), ("restart_3B", (1, 1), "fast")]
# tj3DecodeYUVPlanes8: image sizes (odd, even) and extra bytes per plane row (0: unpitched planes)
DECODE_SIZES = [(7, 5), (16, 10), (227, 149)]
DECODE_PADS = [0, 13]
PIXEL_FORMATS = ["RGB", "BGR", "RGBX", "BGRX", "XBGR", "XRGB", "GRAY", "RGBA", "BGRA", "ABGR", "ARGB", "CMYK"]   # TJPF_* order
PIXEL_SIZE = {"RGB": 3, "BGR": 3, "GRAY": 1}


def decode_cases():
    """[(id, subsampling name, (w, h), pixel format, pad)]"""
    return [(f"dec:{ss}:{w}x{h}:{pf}:{pad}", ss, (w, h), pf, pad) for ss in SUBSAMPS for (w, h) in DECODE_SIZES
            for pf in PIXEL_FORMATS for pad in DECODE_PADS]


def decode_planes(ss, w, h):
    """seeded planes of a TJSAMP_<ss> image of w x h pixels: [(ph, pw) uint8] per plane"""
    si = SUBSAMPS.index(ss)
    rng = np.random.default_rng(si * 100003 + w * 101 + h)
    out = []
    for ci in range(1 if ss == "gray" else 3):
        pw, ph = plane_dims(ci, w, h, si)
        ramp = (np.add.outer(np.arange(ph) * 5, np.arange(pw) * 3) + 60 * ci) % 256
        out.append(np.clip(ramp + rng.integers(-60, 61, (ph, pw)), 0, 255).astype(np.uint8))
    return out


def golden():
    return json.load(open(GOLDEN))


def md5(a) -> str:
    return hashlib.md5(np.ascontiguousarray(a).tobytes()).hexdigest()


def tj_subsamp(info):
    """getSubsamp (turbojpeg.c:400-479) of a parsed source (mozjpeg_b200._abi.SourceInfo), -1 for TJSAMP_UNKNOWN"""
    nc = info.num_components
    h = [info.h_samp_factor[c] for c in range(nc)]; v = [info.v_samp_factor[c] for c in range(nc)]
    cmyk = info.jpeg_color_space in (4, 5)
    if nc == 1 and info.jpeg_color_space == 1:
        return 3
    r = -1
    for i in range(7):
        if i == 3 or not (nc == 3 or (cmyk and nc == 4)):
            continue
        mw, mh = MCU[i][0] // 8, MCU[i][1] // 8
        if (h[0], v[0]) == (mw, mh):
            ref = [(mw, mh) if cmyk and k == 3 else (1, 1) for k in range(1, nc)]
            if all((h[k], v[k]) == ref[k - 1] for k in range(1, nc)):
                return i
        if (h[0], v[0]) == (2, 2) and i in (1, 4):
            ref = [(2, 2) if cmyk and k == 3 else (mh, mw) for k in range(1, nc)]
            if all((h[k], v[k]) == ref[k - 1] for k in range(1, nc)):
                return i
        if h[0] * v[0] <= 10 // 3 and i == 0 and all((h[k], v[k]) == (h[0], v[0]) for k in range(1, nc)):
            r = i                  # the reference's break leaves only its component loop: a later layout may still match
    return r


def plane_dims(ci, w, h, ss):
    """tj3YUVPlaneWidth / tj3YUVPlaneHeight"""
    mw, mh = MCU[ss][0] // 8, MCU[ss][1] // 8
    pw, ph = -(-w // mw) * mw, -(-h // mh) * mh
    return (pw, ph) if ci == 0 else (pw * 8 // MCU[ss][0], ph * 8 // MCU[ss][1])


def plan(info, scale):
    """(TJSAMP_*, [(pw, ph, iw, ih) per plane]) of a source decompressed to planes at ``scale``"""
    ss = tj_subsamp(info)
    k = 8 * scale[0] // scale[1]
    W, H, nc = info.image_width, info.image_height, info.num_components
    hs = [info.h_samp_factor[c] for c in range(nc)]; vs = [info.v_samp_factor[c] for c in range(nc)]
    mh, mv = max(hs), max(vs)
    ow, oh = -(-W * k // 8), -(-H * k // 8)
    out = []
    for c in range(nc):
        wib, hib = -(-W * hs[c] // (mh * 8)), -(-H * vs[c] // (mv * 8))
        out.append((*plane_dims(c, ow, oh, ss), wib * k, hib * k))
    return ss, out


def defined(plane, pw, ph, iw, ih):
    """the samples of a (ph, pw) plane the reference defines: its first min(ih, ph) rows of min(iw, pw)"""
    return plane[:min(ih, ph), :min(iw, pw)]


class RefTJ:
    """The reference's tj3DecompressToYUVPlanes8 (oracle/_ref/libturbojpeg_ref.so), called through ctypes."""

    TJINIT_DECOMPRESS, TJPARAM_SUBSAMP, TJPARAM_FASTDCT = 1, 4, 10

    class ScalingFactor(C.Structure):
        _fields_ = [("num", C.c_int), ("denom", C.c_int)]

    def __init__(self, path=REF_TJ):
        lib = C.CDLL(path)
        lib.tj3Init.argtypes = [C.c_int]; lib.tj3Init.restype = C.c_void_p
        lib.tj3Destroy.argtypes = [C.c_void_p]; lib.tj3Destroy.restype = None
        lib.tj3Set.argtypes = [C.c_void_p, C.c_int, C.c_int]; lib.tj3Set.restype = C.c_int
        lib.tj3Get.argtypes = [C.c_void_p, C.c_int]; lib.tj3Get.restype = C.c_int
        lib.tj3GetErrorStr.argtypes = [C.c_void_p]; lib.tj3GetErrorStr.restype = C.c_char_p
        lib.tj3SetScalingFactor.argtypes = [C.c_void_p, self.ScalingFactor]; lib.tj3SetScalingFactor.restype = C.c_int
        lib.tj3DecompressHeader.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]; lib.tj3DecompressHeader.restype = C.c_int
        lib.tj3YUVPlaneWidth.argtypes = [C.c_int, C.c_int, C.c_int]; lib.tj3YUVPlaneWidth.restype = C.c_int
        lib.tj3YUVPlaneHeight.argtypes = [C.c_int, C.c_int, C.c_int]; lib.tj3YUVPlaneHeight.restype = C.c_int
        lib.tj3YUVBufSize.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]; lib.tj3YUVBufSize.restype = C.c_size_t
        lib.tj3DecompressToYUVPlanes8.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]
        lib.tj3DecompressToYUVPlanes8.restype = C.c_int
        lib.tj3DecodeYUVPlanes8.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.tj3DecodeYUVPlanes8.restype = C.c_int
        lib.tj3CompressFromYUVPlanes8.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p),
                                                  C.POINTER(C.c_size_t)]
        lib.tj3CompressFromYUVPlanes8.restype = C.c_int
        lib.tj3Free.argtypes = [C.c_void_p]; lib.tj3Free.restype = None
        self.lib = lib
        self.h = lib.tj3Init(self.TJINIT_DECOMPRESS)

    def close(self):
        if self.h:
            self.lib.tj3Destroy(self.h)
            self.h = None

    def decompress_planes(self, jpeg: bytes, scale, dct):
        """(TJSAMP_*, [(ph, pw) planes], None), or (None, None, the reference's error)"""
        L = self.lib
        if L.tj3DecompressHeader(self.h, jpeg, len(jpeg)):
            return None, None, L.tj3GetErrorStr(self.h).decode()
        ss = L.tj3Get(self.h, self.TJPARAM_SUBSAMP)
        if L.tj3SetScalingFactor(self.h, self.ScalingFactor(*scale)):
            return None, None, L.tj3GetErrorStr(self.h).decode()
        L.tj3Set(self.h, self.TJPARAM_FASTDCT, int(dct == "fast"))
        w, h = L.tj3Get(self.h, 5), L.tj3Get(self.h, 6)          # TJPARAM_JPEGWIDTH, TJPARAM_JPEGHEIGHT
        ow, oh = -(-w * scale[0] // scale[1]), -(-h * scale[0] // scale[1])   # TJSCALED
        n = 1 if ss == 3 else 3
        bufs = []
        for ci in range(n if 0 <= ss < 7 else 0):
            bufs.append(np.zeros((max(1, L.tj3YUVPlaneHeight(ci, oh, ss)), max(1, L.tj3YUVPlaneWidth(ci, ow, ss))), np.uint8))
        ptrs = (C.c_void_p * 4)(*([b.ctypes.data for b in bufs] + [None] * (4 - len(bufs))))
        if not bufs:
            ptrs[0] = C.cast(C.create_string_buffer(16), C.c_void_p).value
        rc = L.tj3DecompressToYUVPlanes8(self.h, jpeg, len(jpeg), ptrs, None)
        if rc:
            return None, None, L.tj3GetErrorStr(self.h).decode()
        return ss, bufs, None

    def decode_pixels(self, planes, ss, w, h, pf, pad=0):
        """tj3DecodeYUVPlanes8 of one image: ((h, w, pixel size) pixels, None) or (None, the reference's error)"""
        L = self.lib
        L.tj3Set(self.h, self.TJPARAM_SUBSAMP, SUBSAMPS.index(ss))
        bufs = [np.zeros((p.shape[0], p.shape[1] + pad), np.uint8) for p in planes]
        for b, p in zip(bufs, planes):
            b[:, :p.shape[1]] = p
        ptrs = (C.c_void_p * 3)(*([b.ctypes.data for b in bufs] + [None] * (3 - len(bufs))))
        strides = (C.c_int * 3)(*([b.shape[1] for b in bufs] + [0] * (3 - len(bufs)))) if pad else None
        ps = PIXEL_SIZE.get(pf, 4)
        out = np.zeros((h, w, ps), np.uint8)
        if L.tj3DecodeYUVPlanes8(self.h, ptrs, strides, out.ctypes.data, w, 0, h, PIXEL_FORMATS.index(pf)):
            return None, L.tj3GetErrorStr(self.h).decode()
        return out, None

    def recompress(self, jpeg: bytes, scale, dct, quality=75):
        """tj3DecompressToYUVPlanes8 then tj3CompressFromYUVPlanes8 at ``quality`` and the source's subsampling: file bytes"""
        ss, planes, err = self.decompress_planes(jpeg, scale, dct)
        assert err is None, err
        L = self.lib
        c = L.tj3Init(0)                                            # TJINIT_COMPRESS
        try:
            L.tj3Set(c, 3, quality); L.tj3Set(c, self.TJPARAM_SUBSAMP, ss)   # TJPARAM_QUALITY, TJPARAM_SUBSAMP
            ptrs = (C.c_void_p * 3)(*([p.ctypes.data for p in planes] + [None] * (3 - len(planes))))
            buf = C.c_void_p(); size = C.c_size_t(0)
            h, w = planes[0].shape
            ow, oh = self.lib.tj3Get(self.h, 5), self.lib.tj3Get(self.h, 6)
            ow, oh = -(-ow * scale[0] // scale[1]), -(-oh * scale[0] // scale[1])
            if L.tj3CompressFromYUVPlanes8(c, ptrs, ow, None, oh, C.byref(buf), C.byref(size)):
                raise RuntimeError(L.tj3GetErrorStr(c).decode())
            out = C.string_at(buf, size.value)
            L.tj3Free(buf)
            return out
        finally:
            L.tj3Destroy(c)

    def buf_size(self, w, align, h, subsamp):
        return self.lib.tj3YUVBufSize(w, align, h, subsamp)
