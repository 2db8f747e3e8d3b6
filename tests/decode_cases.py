"""Source files of the device-decode tests (tests/test_device_decode.py) and of tools/make_golden.py --decode.

Every source is written by the repository's CPU oracle (bit-identical to the reference's encoder on these inputs), so
a GPU run needs neither the reference's sources nor its binaries; tests/golden/decode_golden.json records the md5 of
each file and of the reference's jpeg_read_coefficients planes for it."""
import hashlib

import numpy as np

# (id, width, height, seed, cjpeg switches, scan layout): "multi" = one sequential scan per component
CASES = [
    ("revert", 200, 136, 1, ["-revert"], None),
    ("revert_optimize", 200, 136, 2, ["-revert", "-optimize"], None),
    ("trellis_1x1", 200, 136, 3, ["-baseline", "-quality", "85", "-sample", "1x1"], None),
    ("sample_3x2", 200, 136, 4, ["-revert", "-sample", "3x2"], None),
    ("sample_422", 200, 136, 5, ["-revert", "-sample", "2x1"], None),
    ("sample_440", 200, 136, 6, ["-revert", "-sample", "1x2"], None),
    ("gray", 200, 136, 7, ["-revert", "-grayscale"], None),
    ("rgb", 200, 136, 8, ["-revert", "-rgb"], None),
    ("restart_1", 200, 136, 9, ["-revert", "-restart", "1"], None),
    ("restart_3B", 200, 136, 10, ["-revert", "-restart", "3B"], None),
    ("q100", 200, 136, 11, ["-revert", "-quality", "100"], None),
    ("q100_noise", 160, 96, -1, ["-revert", "-quality", "100", "-sample", "1x1"], None),
    ("flat", 256, 256, -2, ["-revert"], None),
    ("multi_scan", 200, 136, 12, ["-revert"], "multi"),
    ("multi_scan_restart", 200, 136, 13, ["-revert", "-restart", "2B"], "multi"),
    ("ragged_1x1", 1, 1, 14, ["-revert"], None),
    ("ragged_8x8", 8, 8, 15, ["-revert"], None),
    ("ragged_17x9", 17, 9, 16, ["-revert"], None),
    ("ragged_33x17", 33, 17, 17, ["-revert", "-sample", "2x1"], None),
    ("4k_no_restart", 3840, 2160, 18, ["-revert", "-quality", "90"], None),
    ("4k_restart_1", 3840, 2160, 19, ["-revert", "-quality", "90", "-restart", "1"], None),
]


# Sources built another way (id -> builder in EXTRA below): 12-bit and 4-component files, the coefficient carriers of
# tests/adversarial_cases.py written as plain files, and files edited at the byte or bit level.  Their expected planes
# are only the reference's (decode_golden.json).
EXTRA_IDS = ["baseline12", "ycck", "cmyk", "carrier_fib8_optimize", "carrier_equal8", "carrier_all_symbols8", "carrier_max_magnitude8",
             "carrier_fib12", "carrier_all_symbols12", "carrier_max_magnitude12", "carrier_ff", "carrier_ff_restart",
             "fill_before_rst", "ac_run_past_63", "no_dht"]


def _carrier(planes, precision=8, extra=()):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    hib, wib = planes[0].shape[:2]
    p = mj.params_from_switches((["-precision", "12"] if precision == 12 else []) + ["-revert", *extra], wib * 8, hib * 8, 1)
    return O.oracle_encode_coefs(p, planes)


def _data_range(jpeg: bytes):
    from mozjpeg_b200 import jpegtran as T
    sc = T.parse_source(jpeg).scans[0]
    return sc.data_offset, sc.data_offset + sc.data_size


def _strip_dht(jpeg: bytes) -> bytes:
    """the file without its DHT segments (a reader then uses the standard tables, std_huff_tables)"""
    out, pos = [jpeg[:2]], 2
    while jpeg[pos + 1] != 0xDA:
        ln = int.from_bytes(jpeg[pos + 2:pos + 4], "big")
        if jpeg[pos + 1] != 0xC4:
            out.append(jpeg[pos:pos + 2 + ln])
        pos += 2 + ln
    return b"".join(out) + jpeg[pos:]


def _run_past_63() -> bytes:
    """A gray 16x8 file with the standard tables whose first block codes 49 coefficients of 1 (zigzag 1..49) and then
    the symbol run 15 / size 1, which moves the index to 65: the reference writes the value at position 63 and ends
    the block (jpeg_natural_order's extra entries).  The second block is DC 0 and EOB."""
    from mozjpeg_b200 import jpegtran as T
    base = _carrier([np.zeros((1, 2, 64), np.int16)])
    info = T.parse_source(base)
    sc = info.scans[0]

    def codes(h):
        bits, vals = list(h.bits), list(h.huffval)
        out, code, k = {}, 0, 0
        for l in range(1, 17):
            for _ in range(bits[l]):
                out[vals[k]] = (code, l); code += 1; k += 1
            code <<= 1
        return out

    dc, ac = codes(info.huff[sc.dc_huff[0]]), codes(info.huff[sc.ac_huff[0]])
    bits = []

    def put(v, n):
        bits.extend((v >> (n - 1 - i)) & 1 for i in range(n))

    put(*dc[0])
    for _ in range(49):
        put(*ac[0x01]); put(1, 1)
    put(*ac[0xF1]); put(1, 1)
    put(*dc[0]); put(*ac[0x00])
    bits += [1] * (-len(bits) % 8)
    data = bytearray()
    for i in range(0, len(bits), 8):
        b = int("".join(map(str, bits[i:i + 8])), 2)
        data.append(b)
        if b == 0xFF:
            data.append(0)
    lo, hi = _data_range(base)
    return base[:lo] + bytes(data) + base[hi:]


# coefficient family, precision, extra switches: skewed histograms (16-bit codes), every legal symbol with ZRL chains,
# magnitudes at the coefficient limit; 12-bit files always get optimal tables
_CARRIERS = {"carrier_fib8_optimize": ("fib", 8, ["-optimize"]), "carrier_equal8": ("equal", 8, []),
             "carrier_all_symbols8": ("all_symbols", 8, []), "carrier_max_magnitude8": ("max_magnitude", 8, []),
             "carrier_fib12": ("fib", 12, []), "carrier_all_symbols12": ("all_symbols", 12, []),
             "carrier_max_magnitude12": ("max_magnitude", 12, [])}


def extra_source(name: str) -> bytes:
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    from mozjpeg_b200.synth import synth_image12
    from oracle import oracle as O
    import adversarial_cases as AC
    if name == "baseline12":
        p = mj.params_from_switches(["-precision", "12", "-baseline", "-quality", "75", "-notrellis", "-noovershoot"], 120, 72, 3)
        return O.oracle_encode(p, synth_image12(4, 120, 72)).jpeg
    if name in ("ycck", "cmyk"):
        p = mj.tj3_params(120, 72, quality=85, subsamp="420", cmyk=True, colorspace=A.CS_YCCK if name == "ycck" else A.CS_CMYK)
        px = np.random.default_rng(7).integers(0, 256, (72, 120, 4), dtype=np.uint8)
        px[:, :60] = O.synth_image(8, 60, 72)[..., [0, 1, 2, 0]]
        return O.oracle_encode(p, px).jpeg
    if name.startswith("carrier_ff"):                  # mostly 0xFF bytes: heavy stuffing
        return _carrier(AC.ff_plane(), 8, ["-restart", "1"] if name.endswith("restart") else [])
    if name in _CARRIERS:
        fam, prec, extra = _CARRIERS[name]
        return _carrier(AC.coef_families(prec)[fam], prec, extra)
    if name == "fill_before_rst":                      # fill bytes in front of every fourth RSTn
        import re
        src = extra_source("carrier_ff_restart")
        lo, _ = _data_range(src)
        cut = [m.start() for m in re.finditer(rb"\xff[\xd0-\xd7]", src[lo:])][::4]
        out, prev = [src[:lo]], lo
        for c in cut:
            out += [src[prev:lo + c], b"\xff\xff"]; prev = lo + c
        return b"".join(out) + src[prev:]
    if name == "ac_run_past_63":
        return _run_past_63()
    if name == "no_dht":
        return _strip_dht(source(CASES[0])[0])
    raise KeyError(name)


def pixels(seed: int, w: int, h: int) -> np.ndarray:
    from oracle import oracle as O
    if seed == -1:                                   # noise: long codes, large coefficients
        return np.random.default_rng(5).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if seed == -2:                                   # flat: every block identical, a periodic bit stream
        return np.full((h, w, 3), 97, dtype=np.uint8)
    return O.synth_image(seed, w, h)


def params(case):
    import mozjpeg_b200 as mj
    _, w, h, _, sw, layout = case
    p = mj.params_from_switches(sw, w, h, 3)
    if layout == "multi":
        p.num_scans = p.num_components
        for k in range(p.num_components):
            s = p.scan_info[k]
            s.comps_in_scan, s.Ss, s.Se, s.Ah, s.Al = 1, 0, 63, 0, 0
            s.component_index[0] = k
    return p


def source(case):
    """(file bytes, [per component (hib, wib, 64) int16 natural-order planes the oracle quantized])"""
    from oracle import oracle as O
    _, w, h, seed, _, _ = case
    r = O.oracle_encode(params(case), pixels(seed, w, h), want_debug=True)
    d = r.dbg
    return r.jpeg, [np.ascontiguousarray(d["final"][ci][:d["hib"][ci], :d["wib"][ci]]) for ci in range(d["ncomp"])]


def md5_planes(planes) -> str:
    m = hashlib.md5()
    for a in planes:
        m.update(np.ascontiguousarray(a, dtype=np.int16).tobytes())
    return m.hexdigest()
