"""Sources and expected results of the recompress tests (tests/test_recompress.py) and of tools/make_golden.py
--recompress.

Every source is written by the repository's CPU oracle from seeded images or constructed coefficients, so a GPU run
needs neither the reference's sources nor stored JPEG files; tests/golden/recompress_golden.json records, per source,
the md5 of the file and of the pixels the reference decodes from it (jpeg_read_scanlines of a default decompress
object), and the md5 + size of the reference cjpeg's output for each recompress switch set.

decode_pixels below is a plain numpy restatement of what follows the entropy decode in the reference's decompressor
(jddctmgr.c / jidctint.c, jdsample.c with jdmainct.c's context rows, jdcolor.c).  It is the CPU-side pin of the device
kernels: equal to the recorded md5s everywhere, and to the reference library itself where build/librefdec.so (tests/
refdec.c over oracle/_ref) exists."""
import ctypes as C
import hashlib
import json
import os

import numpy as np

import decode_cases as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "recompress_golden.json")
REFDEC = os.path.join(ROOT, "build", "librefdec.so")
REF_CJPEG = os.path.join(ROOT, "oracle", "_ref", "cjpeg")

# (id, width, height, seed, cjpeg switches of the source, scan layout) -- the tuple format of decode_cases.CASES
CASES = [
    ("s444", 200, 136, 21, ["-revert", "-sample", "1x1"], None),
    ("s422", 200, 136, 22, ["-revert", "-sample", "2x1"], None),
    ("s440", 200, 136, 23, ["-revert", "-sample", "1x2"], None),
    ("s420", 200, 136, 24, ["-revert"], None),
    ("gray", 200, 136, 25, ["-revert", "-grayscale"], None),
    ("rgb", 200, 136, 26, ["-revert", "-rgb"], None),
    # sizes that are no multiple of the iMCU, one pixel wide / high, and 1, 2, 3 downsampled columns
    ("ragged_420", 203, 131, 27, ["-revert"], None),
    ("ragged_422", 33, 17, 28, ["-revert", "-sample", "2x1"], None),
    ("ragged_440", 19, 13, 29, ["-revert", "-sample", "1x2"], None),
    ("ragged_444", 21, 11, 30, ["-revert", "-sample", "1x1"], None),
    ("one_pixel", 1, 1, 31, ["-revert"], None),
    ("one_wide", 1, 37, 32, ["-revert"], None),
    ("one_high", 37, 1, 33, ["-revert"], None),
    ("w2_420", 2, 9, 34, ["-revert"], None),
    ("w3_420", 3, 9, 35, ["-revert"], None),
    ("w4_420", 4, 10, 36, ["-revert"], None),
    ("w5_420", 5, 10, 37, ["-revert"], None),
    ("w6_420", 6, 7, 38, ["-revert"], None),
    ("w2_422", 2, 5, 39, ["-revert", "-sample", "2x1"], None),
    ("w4_422", 4, 5, 40, ["-revert", "-sample", "2x1"], None),
    ("w5_422", 5, 5, 41, ["-revert", "-sample", "2x1"], None),
    ("h2_440", 9, 2, 42, ["-revert", "-sample", "1x2"], None),
    ("h3_440", 9, 3, 43, ["-revert", "-sample", "1x2"], None),
    # taller than a chunk of the smallest size holds blocks for: many iMCU rows
    ("tall", 48, 4100, 44, ["-revert"], None),
    ("q5", 200, 136, 45, ["-revert", "-quality", "5"], None),
    ("q75", 200, 136, 46, ["-revert", "-quality", "75"], None),
    ("q100", 200, 136, 47, ["-revert", "-quality", "100", "-sample", "2x2"], None),
    ("q100_noise", 160, 96, -1, ["-revert", "-quality", "100", "-sample", "2x2"], None),
    ("sof1_dqt16", 200, 136, 48, ["-revert", "-quality", "2"], None),          # table entries above 255: 16-bit DQT, SOF1
    ("restart_1", 200, 136, 49, ["-revert", "-restart", "1"], None),
    ("restart_3B", 203, 131, 50, ["-revert", "-restart", "3B"], None),
    ("multi_scan", 200, 136, 51, ["-revert"], "multi"),
    ("multi_scan_restart", 200, 136, 52, ["-revert", "-restart", "2B", "-sample", "2x1"], "multi"),
]
CASE = {c[0]: c for c in CASES}

# sources built another way: constructed coefficients under flat tables (IDCT_TABLES), and files with extra markers
IDCT_TABLES = {"idct_q1": 1, "idct_q255": 255, "idct_q32767": 32767}
EXTRA_IDS = list(IDCT_TABLES) + ["com_exif"]

COM = b"\xff\xfe" + (2 + 11).to_bytes(2, "big") + b"hello world"
EXIF = b"\xff\xe1" + (2 + 14).to_bytes(2, "big") + b"Exif\0\0MM\0*\0\0\0\x08"

# (source id, cjpeg switches) recompressed by the reference's cjpeg; [] is the library default with its scan search
RECOMPRESS = [(s, sw) for s in ("s420", "ragged_420", "s444") for sw in
              (["-quality", "60"], ["-baseline", "-quality", "75", "-sample", "2x2"], ["-revert", "-progressive"], ["-grayscale"], [])]
RECOMPRESS += [("gray", ["-quality", "60"]), ("gray", []), ("s422", ["-quality", "85"]), ("s440", ["-revert", "-optimize"]),
               ("com_exif", ["-quality", "60"]), ("com_exif", ["-revert", "-nojfif"]),
               ("rgb", ["-revert", "-rgb"]), ("rgb", ["-quality", "60"]), ("multi_scan_restart", ["-revert", "-restart", "1"])]


def idct_planes():
    """One gray component of constructed blocks: each of the 64 basis functions alone at +1023 and -1023, DC-only
    blocks from one clamp to the other, and dense blocks of large random coefficients."""
    rng = np.random.default_rng(11)
    blocks = []
    for k in range(64):
        for a in (1023, -1023):
            b = np.zeros(64, np.int16); b[k] = a; blocks.append(b)
    for dc in np.linspace(-1023, 1023, 32).astype(int):
        b = np.zeros(64, np.int16); b[0] = dc; blocks.append(b)
    for _ in range(32):
        blocks.append(rng.integers(-1023, 1024, 64).astype(np.int16))
    for _ in range(32):
        b = rng.integers(-40, 41, 64).astype(np.int16); b[0] = rng.integers(-1023, 1024); blocks.append(b)
    return [np.stack(blocks).reshape(-1, 32, 64)]


def _insert_after_app0(jpeg: bytes, extra: bytes) -> bytes:
    assert jpeg[2:4] == b"\xff\xe0"
    end = 4 + int.from_bytes(jpeg[4:6], "big")
    return jpeg[:end] + extra + jpeg[end:]


_cache = {}


def source(sid: str):
    """(file bytes, [per component (hib, wib, 64) int16 natural-order planes]) of source ``sid``"""
    if sid in _cache:
        return _cache[sid]
    if sid in CASE:
        r = D.source(CASE[sid])
    elif sid in IDCT_TABLES:
        import mozjpeg_b200 as mj
        from oracle import oracle as O
        planes = idct_planes()
        hib, wib = planes[0].shape[:2]
        p = mj.params_from_switches(["-revert"], wib * 8, hib * 8, 1)
        for k in range(64):
            p.quant_tbl[0][k] = IDCT_TABLES[sid]
        r = (O.oracle_encode_coefs(p, planes), planes)
    elif sid == "com_exif":
        jpeg, planes = source("s420")
        r = (_insert_after_app0(jpeg, COM + EXIF), planes)
    else:
        raise KeyError(sid)
    _cache[sid] = r
    return r


def copied_markers(jpeg: bytes, p) -> bytes:
    """the segments cjpeg re-emits from a JPEG input behind the compressor's own header (cjpeg.c:960-990): the COM and
    APPn segments in front of the first SOS (all sources here are read that far before the copy), without a JFIF APP0 /
    Adobe APP14 the compressor writes itself"""
    out, pos = b"", 2
    while jpeg[pos + 1] != 0xDA:
        m, ln = jpeg[pos + 1], int.from_bytes(jpeg[pos + 2:pos + 4], "big")
        seg, dat = jpeg[pos:pos + 2 + ln], jpeg[pos + 4:pos + 2 + ln]
        dup = (p.write_JFIF_header and m == 0xE0 and dat[:5] == b"JFIF\0") or (p.write_Adobe_marker and m == 0xEE and dat[:5] == b"Adobe")
        if (m == 0xFE or 0xE0 <= m <= 0xEF) and not dup:
            out += seg
        pos += 2 + ln
    return out


def insert_markers(encoded: bytes, markers: bytes) -> bytes:
    """``markers`` behind SOI and the JFIF APP0 / Adobe APP14 segments the file starts with"""
    pos = 2
    while encoded[pos + 1] in (0xE0, 0xEE):
        pos += 2 + int.from_bytes(encoded[pos + 2:pos + 4], "big")
    return encoded[:pos] + markers + encoded[pos:]


def all_ids():
    return [c[0] for c in CASES] + EXTRA_IDS


def golden():
    return json.load(open(GOLDEN))


def md5(b) -> str:
    return hashlib.md5(np.ascontiguousarray(b).tobytes() if isinstance(b, np.ndarray) else b).hexdigest()


# ---------------------------------------------------------------------------------------------- numpy restatement
def _range_limit_table():
    """IDCT_range_limit as prepare_range_limit_table lays it out (jdmaster.c), indexed with (x & RANGE_MASK)"""
    t = np.zeros(1024, np.uint8)
    t[:128] = np.arange(128, 256)          # the upper half of the identity segment
    t[128:512] = 255
    t[512:896] = 0
    t[896:] = np.arange(0, 128)
    return t


def _idct_1d(d, shift):
    """the butterfly of jpeg_idct_islow on eight int64 arrays, descaled by ``shift``"""
    z2, z3 = d[2], d[6]
    z1 = (z2 + z3) * 4433
    tmp2 = z1 - z3 * 15137
    tmp3 = z1 + z2 * 6270
    tmp0 = (d[0] + d[4]) << 13
    tmp1 = (d[0] - d[4]) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = d[7], d[5], d[3], d[1]
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * 9633
    tmp0, tmp1, tmp2, tmp3 = tmp0 * 2446, tmp1 * 16819, tmp2 * 25172, tmp3 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    tmp0, tmp1, tmp2, tmp3 = tmp0 + z1 + z3, tmp1 + z2 + z4, tmp2 + z2 + z3, tmp3 + z1 + z4
    r = 1 << (shift - 1)
    return [(tmp10 + tmp3 + r) >> shift, (tmp11 + tmp2 + r) >> shift, (tmp12 + tmp1 + r) >> shift, (tmp13 + tmp0 + r) >> shift,
            (tmp13 - tmp0 + r) >> shift, (tmp12 - tmp1 + r) >> shift, (tmp11 - tmp2 + r) >> shift, (tmp10 - tmp3 + r) >> shift]


def idct_plane(plane, q):
    """(hib, wib, 64) quantized coefficients, 64 table entries -> (hib * 8, wib * 8) samples"""
    hib, wib = plane.shape[:2]
    qs = np.asarray(q, np.uint16).astype(np.int16).astype(np.int64)            # ISLOW_MULT_TYPE is a short
    d = plane.astype(np.int64).reshape(hib, wib, 8, 8) * qs.reshape(8, 8)
    ws = np.stack(_idct_1d([d[:, :, r, :] for r in range(8)], 11), axis=2).astype(np.int32).astype(np.int64)   # int workspace
    out = np.stack(_idct_1d([ws[:, :, :, c] for c in range(8)], 18), axis=3)
    px = _range_limit_table()[out & 1023]
    return px.transpose(0, 2, 1, 3).reshape(hib * 8, wib * 8)


def _h2_fancy(s, even_bias, odd_bias, shift, edge):
    """the 2:1 horizontal triangle filter over rows of column sums: 3/4 nearer + 1/4 further, first and last output
    from one sum alone"""
    n = s.shape[1]
    out = np.empty((s.shape[0], 2 * n), np.int64)
    out[:, 2::2] = (3 * s[:, 1:] + s[:, :-1] + even_bias) >> shift
    out[:, 1:-1:2] = (3 * s[:, :-1] + s[:, 1:] + odd_bias) >> shift
    out[:, 0] = (s[:, 0] * edge + even_bias) >> shift
    out[:, -1] = (s[:, -1] * edge + odd_bias) >> shift
    return out


def upsample(c, hx, vx, W, H):
    """one chroma plane (padded) -> (H, W): the method jinit_upsampler picks with fancy upsampling on"""
    dw, dh = -(-W // hx), -(-H // vx)
    c = c[:dh, :dw].astype(np.int64)
    if vx == 2 and (hx == 1 or dw > 2):
        # context rows (jdmainct.c): above the first row the first, below the last real row that row
        y = np.arange(2 * dh)
        near = c[y // 2]
        far = c[np.clip(np.where(y % 2 == 0, y // 2 - 1, y // 2 + 1), 0, dh - 1)]
        if hx == 1:                                                      # h1v2_fancy_upsample
            out = (3 * near + far + np.where(y % 2 == 0, 1, 2)[:, None]) >> 2
        else:                                                            # h2v2_fancy_upsample
            out = _h2_fancy(3 * near + far, 8, 7, 4, 4)
    elif hx == 2 and dw > 2:                                             # h2v1_fancy_upsample
        out = _h2_fancy(c, 1, 2, 2, 4)                                   # (4 * s + bias) >> 2 is s: the first and last output copy their sample
    else:                                                                # fullsize / h2v1 / h2v2 replication
        out = np.repeat(np.repeat(c, vx, axis=0), hx, axis=1)
    return out[:H, :W]


def ycc_to_rgb(y, cb, cr):
    """ycc_rgb_convert with the four tables of build_ycc_rgb_table (SCALEBITS 16)"""
    x = np.arange(256, dtype=np.int64) - 128
    cr_r = (91881 * x + 32768) >> 16
    cb_b = (116130 * x + 32768) >> 16
    cr_g = -46802 * x
    cb_g = -22554 * x + 32768
    y = y.astype(np.int64)
    rgb = np.stack([y + cr_r[cr], y + ((cb_g[cb] + cr_g[cr]) >> 16), y + cb_b[cb]], axis=-1)
    return np.clip(rgb, 0, 255).astype(np.uint8)


def decode_pixels(jpeg: bytes, planes):
    """the pixels the reference's decompressor makes of a file whose quantized coefficients are ``planes``"""
    from mozjpeg_b200 import jpegtran as T
    from mozjpeg_b200 import _abi as A
    info = T.parse_source(jpeg)
    W, H, nc = info.image_width, info.image_height, info.num_components
    samples = [idct_plane(np.asarray(planes[c]), list(info.comp_quant[c])) for c in range(nc)]
    if nc == 1:
        return samples[0][:H, :W].copy()
    hx, vx = info.h_samp_factor[0], info.v_samp_factor[0]
    y, cb, cr = samples[0][:H, :W], upsample(samples[1], hx, vx, W, H), upsample(samples[2], hx, vx, W, H)
    if info.jpeg_color_space == A.CS_RGB:
        return np.stack([y, cb, cr], axis=-1).astype(np.uint8)
    return ycc_to_rgb(y, cb, cr)


# ---------------------------------------------------------------------------------------------- the reference
def have_reference() -> bool:
    return os.path.exists(REFDEC) and os.path.exists(REF_CJPEG)


_lib = None


def ref_decompress(jpeg: bytes, header_only: bool = False):
    """(pixels, info) from the unmodified reference library: info = width, height, output_components,
    out_color_space, jpeg_color_space, warnings"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(REFDEC)
        _lib.refdec_decompress.argtypes = [C.c_char_p, C.c_ulong, C.c_void_p, C.c_ulong, C.POINTER(C.c_int)]
        _lib.refdec_decompress.restype = C.c_int
    info = (C.c_int * 6)()
    if _lib.refdec_decompress(jpeg, len(jpeg), None, 0, info):
        raise RuntimeError("the reference refuses the file")
    if header_only:
        return None, list(info)
    w, h, nc = info[0], info[1], info[2]
    out = np.empty((h, w, nc), np.uint8)
    if _lib.refdec_decompress(jpeg, len(jpeg), out.ctypes.data, out.size, info):
        raise RuntimeError("the reference refuses the file")
    return (out[..., 0] if nc == 1 else out), list(info)


def ref_cjpeg(jpeg: bytes, switches) -> bytes:
    """``cjpeg <switches>`` of the reference reading the JPEG file from stdin"""
    import subprocess
    r = subprocess.run([REF_CJPEG, *switches], input=jpeg, capture_output=True)
    if r.returncode != 0:
        raise RuntimeError("reference cjpeg failed: " + r.stderr.decode(errors="replace"))
    return r.stdout
