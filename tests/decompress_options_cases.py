"""Sources, option sets and expected results of the decompress-options tests (tests/test_decompress_options.py) and of
tools/make_golden.py --decompress-options.

Every source is written by the repository's CPU oracle (tests/recompress_cases.py, tests/decode_cases.py), so a GPU
run needs no stored JPEG file.  tests/golden/decompress_options_golden.json records per (source, options) the md5 of
the source and what the reference's decompressor reports and produces with those options set before
jpeg_start_decompress (tests/refdecopt.c): output size, out_color_space, output_components, per component
DCT_scaled_size and downsampled size, and the md5 of the pixels.

plan() below restates jpeg_calc_output_dimensions and the upsampler choice of jinit_upsampler; it is checked against
the recorded fields on the CPU."""
import ctypes as C
import json
import os

import numpy as np

import decode_cases as D
import recompress_cases as R

ROOT = R.ROOT
GOLDEN = os.path.join(ROOT, "tests", "golden", "decompress_options_golden.json")
REFDECOPT = os.path.join(ROOT, "build", "librefdecopt.so")

DCT = {"int": 0, "fast": 1, "float": 2}
CS = {"gray": 1, "rgb": 2, "ycbcr": 3, "ext_rgb": 6, "rgbx": 7, "bgr": 8, "bgrx": 9, "xbgr": 10, "xrgb": 11, "rgba": 12,
      "bgra": 13, "abgr": 14, "argb": 15}

# one ragged size per layout (decode_cases tuple format)
LAYOUTS = [
    ("o_gray", 227, 149, 61, ["-revert", "-grayscale"], None),
    ("o_444", 227, 149, 62, ["-revert", "-sample", "1x1"], None),
    ("o_422", 227, 149, 63, ["-revert", "-sample", "2x1"], None),
    ("o_440", 227, 149, 64, ["-revert", "-sample", "1x2"], None),
    ("o_420", 227, 149, 65, ["-revert"], None),
    ("o_rgb", 227, 149, 66, ["-revert", "-rgb"], None),
]
FOURK = ("o_4k", 3840, 2160, 67, ["-revert", "-quality", "90", "-sample", "2x2"], None)
_LAYOUT = {c[0]: c for c in LAYOUTS + [FOURK]}

SCALES = [(1, 8), (1, 4), (1, 2), (1, 1)]


def case_id(sid, scale, dct, fancy, cs):
    return f"{sid}:{scale[0]}/{scale[1]}:{dct}:{'fancy' if fancy else 'nofancy'}:{cs or 'default'}"


def cases():
    """[(id, source id, (num, denom), dct, fancy, colorspace name or None)]"""
    out = []

    def add(sid, scale, dct="int", fancy=True, cs=None):
        cid = case_id(sid, scale, dct, fancy, cs)
        if cid not in {c[0] for c in out}:
            out.append((cid, sid, scale, dct, fancy, cs))
    # every layout x scale x method x fancy
    for lay in LAYOUTS:
        for sc in SCALES:
            for dct in DCT:
                for fancy in (True, False):
                    add(lay[0], sc, dct, fancy)
    # output colour spaces, each at two layouts (the merged upsampler: 2x1 / 2x2 luma, fancy off, equal scaled sizes)
    for cs in CS:
        add("o_420", (1, 2), "int", True, cs)
        add("o_422", (1, 1), "int", False, cs)
    for cs in ("gray", "rgb", "rgbx", "bgr", "argb"):
        add("o_gray", (1, 4), "fast", True, cs)
    for cs in ("gray", "rgb", "bgrx", "xbgr"):
        add("o_rgb", (1, 2), "float", True, cs)
    add("o_420", (1, 1), "int", False, "bgra")                  # merged h2v2
    # small sizes: 1 .. 3 samples of chroma at every scale
    for sid in ("one_pixel", "one_wide", "one_high", "w2_420", "w3_420", "w5_420", "w6_420", "w2_422", "w4_422", "w5_422",
                "h2_440", "h3_440", "ragged_444"):
        for sc in SCALES[:3]:
            for fancy in (True, False):
                add(sid, sc, "int", fancy)
    # content: quality ladder, 16-bit DQT, constructed blocks under flat tables of 1, 255 and 32767, restarts
    for sid in ("q5", "q100", "q100_noise", "sof1_dqt16", "idct_q1", "idct_q255", "idct_q32767", "restart_1", "restart_3B", "multi_scan"):
        for sc in SCALES:
            for dct in DCT:
                add(sid, sc, dct, True)
    # fractions bucketed by the reference (1/5 -> 2/8, 3/16 -> 2/8, 3/7 -> 4/8), and one 4K frame
    add("o_420", (1, 5)); add("o_422", (3, 16), "fast"); add("o_444", (3, 7), "float", False)
    add("o_4k", (1, 4)); add("o_4k", (1, 8), "int", False)
    return out


# scale fractions the device refuses (block sizes 3, 5, 6, 7, 9 .. 16) and colour pairs the reference refuses
REFUSED_SCALES = [(3, 8), (5, 8), (6, 8), (7, 8), (9, 8), (2, 1), (3, 2)]
REFUSED_PAIRS = [("o_gray", 3), ("o_rgb", 3), ("o_420", 0), ("o_gray", 0)]      # (source, out_color_space)
UNSUPPORTED_CS = [4, 5, 16]                                                      # CMYK, YCCK, RGB565 output


def source(sid):
    if sid in _LAYOUT:
        if sid not in R._cache:
            R._cache[sid] = D.source(_LAYOUT[sid])
        return R._cache[sid]
    return R.source(sid)


def golden():
    return json.load(open(GOLDEN))


md5 = R.md5


def opts_tuple(scale, dct, fancy, cs):
    return (scale[0], scale[1], DCT[dct], int(bool(fancy)), -1 if cs is None else CS[cs])


def block_size(num, denom):
    """the IDCT block size jpeg_core_output_dimensions picks for scale_num / scale_denom"""
    for k in range(1, 16):
        if num * 8 <= denom * k:
            return k
    return 16


def plan(info, scale, fancy):
    """(output width, height, [per component (DCT_scaled_size, downsampled_width, downsampled_height, upsampler)]) for
    a parsed source: jpeg_calc_output_dimensions (jdmaster.c) and the method jinit_upsampler picks (jdsample.c)"""
    k = block_size(*scale)
    W, H, nc = info.image_width, info.image_height, info.num_components
    hs = [info.h_samp_factor[c] for c in range(nc)]; vs = [info.v_samp_factor[c] for c in range(nc)]
    mh, mv = max(hs), max(vs)
    comps = []
    for c in range(nc):
        ss = k
        while ss < 8 and (mh * k) % (hs[c] * ss * 2) == 0 and (mv * k) % (vs[c] * ss * 2) == 0:
            ss *= 2
        dw = -(-W * hs[c] * ss // (mh * 8)); dh = -(-H * vs[c] * ss // (mv * 8))
        hr, vr = mh // (hs[c] * ss // k), mv // (vs[c] * ss // k)
        do_fancy = fancy and k > 1
        up = "fullsize" if (hr, vr) == (1, 1) else \
             ("h2v1_fancy" if do_fancy and dw > 2 else "h2v1") if (hr, vr) == (2, 1) else \
             ("h1v2_fancy" if do_fancy else "int") if (hr, vr) == (1, 2) else \
             ("h2v2_fancy" if do_fancy and dw > 2 else "h2v2")
        comps.append((ss, dw, dh, up))
    return -(-W * k // 8), -(-H * k // 8), comps


def have_reference() -> bool:
    return os.path.exists(REFDECOPT)


_lib = None


def ref_decompress(jpeg: bytes, opts, header_only: bool = False):
    """(pixels or None, info, message) from the unmodified reference library with opts (opts_tuple) set; info as
    tests/refdecopt.c lays it out; pixels None and message set when the library refuses"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(REFDECOPT)
        _lib.refdecopt_decompress.argtypes = [C.c_char_p, C.c_ulong, C.POINTER(C.c_int), C.c_void_p, C.c_ulong, C.POINTER(C.c_int), C.c_char_p]
        _lib.refdecopt_decompress.restype = C.c_int
    o = (C.c_int * 5)(*opts)
    info = (C.c_int * 20)()
    msg = C.create_string_buffer(200)
    if _lib.refdecopt_decompress(jpeg, len(jpeg), o, None, 0, info, msg):
        return None, list(info), msg.value.decode()
    if header_only:
        return None, list(info), ""
    w, h, nc = info[0], info[1], info[2]
    out = np.empty((h, w, nc), np.uint8)
    if _lib.refdecopt_decompress(jpeg, len(jpeg), o, out.ctypes.data, out.size, info, msg):
        return None, list(info), msg.value.decode()
    return (out[..., 0] if nc == 1 else out), list(info), ""
