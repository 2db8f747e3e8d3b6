"""Sources, option sets and expected results of the CMYK / YCCK decompress tests (tests/test_cmyk_decode.py) and of
tools/make_golden.py --cmyk.

Every source is written by the repository's CPU oracle (tests/colorspace_cases.py oracle_encode, which gives YCCK files
the reference's conversion and APP14 transform value), so a GPU run needs no stored JPEG file.
tests/golden/cmyk_golden.json records per (source, options) the md5 of the source and what the reference's
decompressor reports and produces with those options (tests/refdecopt.c): output size, out_color_space,
output_components, per component DCT_scaled_size and downsampled size, and the md5 of the pixels; the refused colour
pairs with the reference's message; and per recompress case the size and md5 of the reference cjpeg's output."""
import json
import os

import numpy as np

import colorspace_cases as CS
import decompress_options_cases as O
import recompress_cases as R

ROOT = R.ROOT
GOLDEN = os.path.join(ROOT, "tests", "golden", "cmyk_golden.json")
CMYK, YCCK = 4, 5

# (id, width, height, seed, TJSAMP name or explicit factors per component, J_COLOR_SPACE, extra): extra "restart",
# "multi" (one sequential scan per component), "dqt16" (table entries above 255: 16-bit DQT, SOF1), "prog"
SOURCES = [
    ("cmyk_444", 227, 149, 1, "444", CMYK, None),
    ("cmyk_420", 227, 149, 2, "420", CMYK, None),
    ("ycck_420", 227, 149, 3, "420", YCCK, None),
    ("ycck_422", 227, 149, 4, "422", YCCK, None),
    ("ycck_440", 227, 149, 5, "440", YCCK, None),
    ("ycck_444", 227, 149, 6, "444", YCCK, None),
    # jpeg_set_colorspace(JCS_YCCK)'s own layout (jcparam.c): 2x2, 1x1, 1x1, 2x2
    ("ycck_libjpeg", 131, 77, 7, None, YCCK, None),
    # K subsampled under full-size C, M, Y: component 0 is not the largest
    ("cmyk_k_sub", 97, 61, 8, ((1, 1), (1, 1), (1, 1), (2, 2)), CMYK, None),
    ("ycck_1x1", 1, 1, 9, "420", YCCK, None),
    ("ycck_w1", 1, 19, 10, "420", YCCK, None),
    ("ycck_w2", 2, 19, 11, "420", YCCK, None),
    ("ycck_w3", 3, 19, 12, "420", YCCK, None),
    ("ycck_w5", 5, 21, 13, "420", YCCK, None),       # 3 subsampled columns
    ("ycck_w4_422", 4, 9, 14, "422", YCCK, None),    # 2 subsampled columns
    ("ycck_h1", 23, 1, 15, "440", YCCK, None),
    ("ycck_h2", 23, 2, 16, "440", YCCK, None),
    ("ycck_h3", 23, 3, 17, "420", YCCK, None),
    ("cmyk_restart", 131, 77, 18, "420", CMYK, "restart"),
    ("ycck_restart", 131, 77, 19, "422", YCCK, "restart"),
    ("ycck_multi", 131, 77, 20, "420", YCCK, "multi"),
    ("cmyk_dqt16", 131, 77, 21, "444", CMYK, "dqt16"),
    ("cmyk_prog", 131, 77, 22, "420", CMYK, "prog"),
    ("ycck_prog", 131, 77, 23, "420", YCCK, "prog"),
]
_SRC = {s[0]: s for s in SOURCES}
SCALES = [(1, 8), (1, 4), (1, 2), (1, 1)]


def case_id(sid, scale, dct, fancy, cs):
    return O.case_id(sid, scale, dct, fancy, cs)


def cases():
    """[(id, source id, (num, denom), dct, fancy, colorspace: None, "cmyk" or "ycck")]; the scales 3/4 and 2/1 need
    all_scales"""
    out = []

    def add(sid, scale, dct="int", fancy=True, cs=None):
        cid = case_id(sid, scale, dct, fancy, cs)
        if cid not in {c[0] for c in out}:
            out.append((cid, sid, scale, dct, fancy, cs))
    for sid in ("cmyk_444", "cmyk_420", "ycck_420", "ycck_422", "ycck_440", "ycck_444"):
        for sc in SCALES:
            for dct in O.DCT:
                for fancy in (True, False):
                    add(sid, sc, dct, fancy)
        add(sid, (3, 4)); add(sid, (2, 1)); add(sid, (2, 1), "int", False)
    for sid in ("ycck_libjpeg", "cmyk_k_sub"):
        for sc in SCALES + [(3, 4), (2, 1)]:
            for fancy in (True, False):
                add(sid, sc, "int", fancy)
    for sid in ("ycck_1x1", "ycck_w1", "ycck_w2", "ycck_w3", "ycck_w5", "ycck_w4_422", "ycck_h1", "ycck_h2", "ycck_h3"):
        for sc in SCALES:
            for fancy in (True, False):
                add(sid, sc, "int", fancy)
    for sid in ("cmyk_restart", "ycck_restart", "ycck_multi", "cmyk_dqt16", "cmyk_prog", "ycck_prog"):
        for sc in ((1, 4), (1, 1)):
            for dct in O.DCT:
                add(sid, sc, dct, True)
    # explicit output colour spaces: CMYK of both kinds, YCCK of a YCCK file
    for sid in ("cmyk_444", "ycck_420", "ycck_libjpeg"):
        add(sid, (1, 1), "int", True, "cmyk")
        add(sid, (1, 2), "fast", False, "cmyk")
    for sid in ("ycck_420", "ycck_422", "ycck_prog"):
        add(sid, (1, 1), "int", True, "ycck")
        add(sid, (1, 4), "float", True, "ycck")
    return out


def needs_all_scales(scale):
    return O.block_size(*scale) not in (1, 2, 4, 8)


def opts(scale, dct, fancy, cs):
    """decompress keywords of a case, with cmyk on"""
    kw = dict(scale=scale, dct=dct, fancy=fancy, colorspace=cs, cmyk=True)
    if needs_all_scales(scale):
        kw["all_scales"] = True
    return kw


def opts_tuple(scale, dct, fancy, cs):
    return (scale[0], scale[1], O.DCT[dct], int(bool(fancy)), {None: -1, "cmyk": CMYK, "ycck": YCCK}[cs])


# colour pairs the reference refuses with "Unsupported color conversion request": (source, out_color_space)
REFUSED_PAIRS = [("cmyk_444", 1), ("cmyk_444", 2), ("ycck_420", 1), ("ycck_420", 2), ("ycck_420", 3), ("ycck_420", 6),
                 ("ycck_420", 12), ("cmyk_420", YCCK), ("o_gray", CMYK), ("o_420", CMYK), ("o_rgb", CMYK), ("o_gray", YCCK),
                 ("o_420", YCCK)]

# recompress cases: (id, source id, cjpeg switches); the "adobe" and "markers" sources are cmyk_420 / ycck_420 with
# extra segments
RECOMPRESS = [
    ("cmyk_444:q75", "cmyk_444", ["-quality", "75"]),
    ("cmyk_420:baseline_q90", "cmyk_420", ["-baseline", "-quality", "90"]),
    ("ycck_420:q75", "ycck_420", ["-quality", "75"]),
    ("ycck_422:baseline_q90", "ycck_422", ["-baseline", "-quality", "90"]),
    ("ycck_libjpeg:revert", "ycck_libjpeg", ["-revert"]),
    ("cmyk_restart:q50_restart", "cmyk_restart", ["-quality", "50", "-restart", "2"]),
    ("ycck_prog:q75", "ycck_prog", ["-quality", "75"]),
    ("ycck_markers:q75", "ycck_markers", ["-quality", "75"]),
    ("cmyk_markers:baseline_q90", "cmyk_markers", ["-baseline", "-quality", "90"]),
]

_cache = {}


def _params(c):
    import mozjpeg_b200 as mj
    sid, w, h, seed, samp, cs, extra = c
    if samp is None:                                   # jpeg_set_colorspace's sampling
        p = mj.tj3_params(w, h, quality=88, subsamp="444", cmyk=True, colorspace=cs)
        p.comp_info[0].h_samp_factor = p.comp_info[0].v_samp_factor = 2
        p.comp_info[3].h_samp_factor = p.comp_info[3].v_samp_factor = 2
    elif isinstance(samp, str):
        p = mj.tj3_params(w, h, quality=80 + seed % 15, subsamp=samp, progressive=extra == "prog", cmyk=True, colorspace=cs)
    else:
        p = mj.tj3_params(w, h, quality=85, subsamp="444", cmyk=True, colorspace=cs)
        for ci, (hh, vv) in enumerate(samp):
            p.comp_info[ci].h_samp_factor, p.comp_info[ci].v_samp_factor = hh, vv
    if extra == "restart":
        p.restart_interval = 1
    elif extra == "multi":
        p.num_scans = p.num_components
        for k in range(p.num_components):
            s = p.scan_info[k]
            s.comps_in_scan, s.Ss, s.Se, s.Ah, s.Al = 1, 0, 63, 0, 0
            s.component_index[0] = k
    elif extra == "dqt16":
        for t in range(2):
            for k in range(64):
                p.quant_tbl[t][k] = 40 + 9 * k            # up to 607
    return p


def source(sid: str) -> bytes:
    """the file bytes of source ``sid`` (SOURCES, the markers variants, or a decompress_options_cases layout)"""
    if sid in _cache:
        return _cache[sid]
    if sid in _SRC:
        c = _SRC[sid]
        jpeg = CS.oracle_encode(_params(c), CS.cmyk_image(c[3], c[1], c[2])).jpeg
    elif sid in ("cmyk_markers", "ycck_markers"):
        base = source(sid.replace("markers", "420"))
        # a COM and an APP2 behind the Adobe APP14 the file starts with
        jpeg = R.insert_markers(base, b"\xff\xfe\x00\x0bCMYK test" + b"\xff\xe2\x00\x0aICC-ish\x00")
    else:
        return O.source(sid)[0]
    _cache[sid] = jpeg
    return jpeg


def source_planes(sid: str):
    """the quantized coefficient planes of source ``sid`` as the oracle wrote them, [per component (hib, wib, 64)]"""
    c = _SRC[sid]
    d = CS.oracle_encode(_params(c), CS.cmyk_image(c[3], c[1], c[2]), want_debug=True).dbg
    return [np.ascontiguousarray(d["final"][ci][:d["hib"][ci], :d["wib"][ci]]) for ci in range(d["ncomp"])]


def golden():
    return json.load(open(GOLDEN))


md5 = R.md5


# ycck_cmyk_convert (jdcolor.c:544-587) with the build_ycc_rgb_table terms (SCALEBITS 16): C, M, Y =
# range_limit[255 - (Y + term)], K passes through
def ycck_to_cmyk(ycck: np.ndarray) -> np.ndarray:
    a = ycck.astype(np.int64)
    y, cb, cr = a[..., 0], a[..., 1] - 128, a[..., 2] - 128
    out = np.empty_like(ycck)
    out[..., 0] = np.clip(255 - (y + ((91881 * cr + 32768) >> 16)), 0, 255)
    out[..., 1] = np.clip(255 - (y + ((-22554 * cb - 46802 * cr + 32768) >> 16)), 0, 255)
    out[..., 2] = np.clip(255 - (y + ((116130 * cb + 32768) >> 16)), 0, 255)
    out[..., 3] = ycck[..., 3]
    return out
