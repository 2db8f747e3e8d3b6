"""Source files of the progressive-decode tests (tests/test_progressive_decode.py) and of tools/make_golden.py
--progressive, and a restatement of the reference's progression checks.

Every source is written by the repository's CPU oracle (bit-identical to the reference's encoder on these inputs), then
edited at the byte level where a case needs it, so a GPU run needs neither the reference's sources nor its binaries;
tests/golden/progressive_golden.json records per source the md5 of the file, of the reference's
jpeg_read_coefficients planes, of its jpegtran outputs and of its default decompression, or the reference's refusal."""
import hashlib
import os
import struct
import tempfile

import numpy as np

from common import GOLD

# (id, width, height, seed, cjpeg switches)
CASES = [
    ("default_q30", 200, 136, 1, ["-quality", "30"]),
    ("default_q75", 200, 136, 2, ["-quality", "75"]),
    ("default_q95", 200, 136, 3, ["-quality", "95"]),
    ("progressive", 200, 136, 4, ["-progressive"]),
    ("progressive_revert", 200, 136, 5, ["-progressive", "-revert"]),
    ("dc_scan_opt0", 200, 136, 6, ["-dc-scan-opt", "0"]),
    ("dc_scan_opt1", 200, 136, 7, ["-dc-scan-opt", "1"]),
    ("dc_scan_opt2", 200, 136, 8, ["-dc-scan-opt", "2"]),
    ("scans_a", 200, 136, 9, ["-scans", "@GOLD/scans_a.txt"]),
    ("scans_b", 200, 136, 10, ["-scans", "@GOLD/scans_b.txt"]),
    ("scans_c", 200, 136, 11, ["-scans", "@GOLD/scans_c.txt"]),
    ("al_chain", 200, 136, 12, ["-scans", "@AL_CHAIN"]),
    ("sample_420", 200, 136, 13, ["-revert", "-progressive", "-sample", "2x2"]),
    ("sample_422", 200, 136, 14, ["-revert", "-progressive", "-sample", "2x1"]),
    ("sample_440", 200, 136, 15, ["-revert", "-progressive", "-sample", "1x2"]),
    ("sample_3x2", 200, 136, 16, ["-revert", "-progressive", "-sample", "3x2"]),
    ("gray", 200, 136, 17, ["-grayscale"]),
    ("rgb", 200, 136, 18, ["-rgb"]),
    ("restart_1", 200, 136, 19, ["-revert", "-progressive", "-restart", "1"]),
    ("restart_3B", 200, 136, 20, ["-revert", "-progressive", "-restart", "3B"]),
    ("default_restart_1", 200, 136, 21, ["-restart", "1"]),
    ("ragged_1x1", 1, 1, 22, []),
    ("ragged_17x9", 17, 9, 23, ["-revert", "-progressive"]),
    ("ragged_33x17", 33, 17, 24, ["-revert", "-progressive", "-sample", "2x1"]),
    ("4k_q75", 3840, 2160, 25, ["-revert", "-progressive", "-quality", "75"]),
]

# a script with Al chains down from 5 and split bands (DC refinements at four levels, AC bands refined three times)
AL_CHAIN = """0 1 2: 0-0, 0, 5;
0: 1-5, 0, 3;
0: 6-63, 0, 4;
1: 1-63, 0, 2;
2: 1-63, 0, 2;
0 1 2: 0-0, 5, 4;
0: 6-63, 4, 3;
0: 1-5, 3, 2;
0: 6-63, 3, 2;
0 1 2: 0-0, 4, 3;
1: 1-63, 2, 1;
0: 1-63, 2, 1;
0 1 2: 0-0, 3, 2;
0 1 2: 0-0, 2, 1;
2: 1-63, 2, 1;
0 1 2: 0-0, 1, 0;
2: 1-63, 1, 0;
0: 1-63, 1, 0;
1: 1-63, 1, 0;
"""

# built another way: 12-bit, 4-component, the coefficient carriers of tests/adversarial_cases.py, and byte-level edits
EXTRA_IDS = ["prog12", "cmyk", "ycck", "carrier_fib8", "carrier_all_symbols8", "carrier_max_magnitude8", "carrier_all_symbols12",
             "carrier_eobrun", "carrier_eobrun_restart", "carrier_corrections",
             "drop_to_dc_only", "drop_last_refinement", "drop_chroma_ac",
             "swap_scans", "wrong_ah", "ac_before_dc", "two_component_ac", "truncated", "corrupt",
             "eobrun_past_restart", "al_14", "two_component_ac_tables"]


def _switches(sw):
    out = []
    for s in sw:
        if s.startswith("@GOLD/"):
            s = os.path.join(GOLD, s[6:])
        elif s == "@AL_CHAIN":
            f = tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False)
            f.write(AL_CHAIN); f.close()
            s = f.name
        out.append(s)
    return out


def source(case) -> bytes:
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    _, w, h, seed, sw = case
    args = _switches(sw)
    try:
        p = mj.params_from_switches(args, w, h, 3)
    finally:
        if "@AL_CHAIN" in sw:
            os.unlink(args[sw.index("@AL_CHAIN")])
    return O.oracle_encode(p, O.synth_image(seed, w, h)).jpeg


def _carrier(planes, precision=8, extra=()):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    hib, wib = planes[0].shape[:2]
    p = mj.params_from_switches((["-precision", "12"] if precision == 12 else []) + ["-revert", "-progressive", *extra], wib * 8, hib * 8, 1)
    return O.oracle_encode_coefs(p, planes)


def segments(jpeg: bytes):
    """[(marker, start, end)] of every marker segment, an SOS's entropy-coded data included in its segment"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(jpeg)
    data = {s.data_offset: s.data_offset + s.data_size for s in info.scans}
    out, pos = [], 2
    while pos + 4 <= len(jpeg) and jpeg[pos + 1] != 0xD9:
        m, ln = jpeg[pos + 1], struct.unpack(">H", jpeg[pos + 2:pos + 4])[0]
        end = pos + 2 + ln
        if m == 0xDA:
            end = data[end]
        out.append((m, pos, end))
        pos = end
    return out


def sos_params(jpeg: bytes):
    """per SOS segment: (component indices, Ss, Se, Ah, Al)"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(jpeg)
    return [(tuple(s.component_index[i] for i in range(s.comps_in_scan)), s.Ss, s.Se, s.Ah, s.Al) for s in info.scans]


def _keep_scans(jpeg: bytes, keep) -> bytes:
    segs = segments(jpeg)
    sos = [k for k, s in enumerate(segs) if s[0] == 0xDA]
    drop = {sos[i] for i in range(len(sos)) if not keep(i)}
    return jpeg[:2] + b"".join(jpeg[a:b] for k, (m, a, b) in enumerate(segs) if k not in drop) + b"\xff\xd9"


def _swap_scans(jpeg: bytes, i: int, j: int) -> bytes:
    segs = segments(jpeg)
    sos = [k for k, s in enumerate(segs) if s[0] == 0xDA]
    order = list(range(len(segs)))
    order[sos[i]], order[sos[j]] = order[sos[j]], order[sos[i]]
    return jpeg[:2] + b"".join(jpeg[segs[k][1]:segs[k][2]] for k in order) + b"\xff\xd9"


def _sos_byte(jpeg: bytes, scan: int, field: str, value: int) -> bytes:
    """the file with one SOS header field (Ss, Se, or Ah/Al byte) set"""
    segs = [s for s in segments(jpeg) if s[0] == 0xDA]
    _, a, _ = segs[scan]
    ns = jpeg[a + 4]
    off = a + 5 + 2 * ns + {"Ss": 0, "Se": 1, "AhAl": 2}[field]
    return jpeg[:off] + bytes([value]) + jpeg[off + 1:]


def _huff_codes(h):
    """{symbol: (code, length)} of a b200jpeg_huff_tbl"""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(h.bits[ln]):
            out[h.huffval[k]] = (code, ln); code += 1; k += 1
        code <<= 1
    return out


def _eobrun_past_restart() -> bytes:
    """A gray progressive file with restarts every block row whose AC bands are all zero, so each restart segment of an
    AC scan is one EOBr symbol for the row's 25 blocks (r = 4, appended bits 9).  The appended bits are set to 15: every
    run now claims 31 blocks and overshoots its segment, which the reference ignores (EOBRUN restarts at each RSTn)."""
    import re
    from mozjpeg_b200 import jpegtran as T
    plane = np.zeros((4, 25, 64), np.int16)
    plane[..., 0] = (np.arange(100).reshape(4, 25) % 7) * 5 - 15
    jpeg = _carrier([plane], 8, ["-restart", "1"])
    info = T.parse_source(jpeg)
    out, prev = [], 0
    for sc in info.scans:
        if sc.Ss == 0:
            continue
        codes = {v: k for k, v in _huff_codes(info.huff[sc.ac_huff[0]]).items()}
        lo, hi = sc.data_offset, sc.data_offset + sc.data_size
        pieces = re.split(rb"(\xff[\xd0-\xd7])", jpeg[lo:hi])
        for k in range(0, len(pieces), 2):
            data = pieces[k].replace(b"\xff\x00", b"\xff")
            bits = "".join(f"{b:08b}" for b in data)
            sym = next(sym for (c, ln), sym in codes.items() if bits[:ln] == format(c, f"0{ln}b"))
            ln = next(ln for (c, ln), v in codes.items() if v == sym)
            r = sym >> 4
            assert sym & 15 == 0 and 0 < r < 15, sym
            bits = bits[:ln] + "1" * r + bits[ln + r:]
            data = bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))
            pieces[k] = data.replace(b"\xff", b"\xff\x00")
        out += [jpeg[prev:lo], b"".join(pieces)]
        prev = hi
    return b"".join(out) + jpeg[prev:]


def extra_source(name: str) -> bytes:
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    from mozjpeg_b200.synth import synth_image12
    from oracle import oracle as O
    import adversarial_cases as AC
    if name == "prog12":
        p = mj.params_from_switches(["-precision", "12", "-revert", "-progressive", "-quality", "75", "-notrellis", "-noovershoot"], 120, 72, 3)
        return O.oracle_encode(p, synth_image12(4, 120, 72)).jpeg
    if name in ("ycck", "cmyk"):
        p = mj.tj3_params(120, 72, quality=85, subsamp="420", progressive=True, cmyk=True, colorspace=A.CS_YCCK if name == "ycck" else A.CS_CMYK)
        px = np.random.default_rng(7).integers(0, 256, (72, 120, 4), dtype=np.uint8)
        px[:, :60] = O.synth_image(8, 60, 72)[..., [0, 1, 2, 0]]
        return O.oracle_encode(p, px).jpeg
    if name == "eobrun_past_restart":
        return _eobrun_past_restart()
    if name.startswith("carrier_eobrun"):          # long EOB runs (up to 0x7FFF blocks), with and without restarts
        return _carrier(AC.eobrun_plane(65536), 8, ["-restart", "7"] if name.endswith("restart") else [])
    if name == "carrier_corrections":              # refinement blocks that carry many correction bits
        f = tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False)
        f.write(AC.REFINE_SCANS); f.close()
        planes = AC.correction_plane()
        hib, wib = planes[0].shape[:2]
        try:
            p = mj.params_from_switches(["-revert", "-scans", f.name], wib * 8, hib * 8, 1)
        finally:
            os.unlink(f.name)
        return O.oracle_encode_coefs(p, planes)
    if name.startswith("carrier_"):
        fam, prec = name[len("carrier_"):-1 if name.endswith("8") else -2], 8 if name.endswith("8") else 12
        return _carrier(AC.coef_families(prec)[fam], prec)
    base = source(CASES[1])                            # the default profile at q75
    prm = sos_params(base)
    if name == "drop_to_dc_only":
        return _keep_scans(base, lambda i: prm[i][1] == 0 and prm[i][3] == 0)
    if name == "drop_last_refinement":
        last = max(i for i, s in enumerate(prm) if s[3] > 0 and s[1] > 0)
        return _keep_scans(base, lambda i: i != last)
    if name == "drop_chroma_ac":
        return _keep_scans(base, lambda i: not (prm[i][1] > 0 and prm[i][0][0] != 0))
    if name == "swap_scans":                           # a refinement in front of its first scan: Ah differs
        ref = next(i for i, s in enumerate(prm) if s[3] > 0 and s[1] > 0)
        first = max(i for i in range(ref) if prm[i][0] == prm[ref][0] and prm[i][1] <= prm[ref][1] <= prm[i][2])
        return _swap_scans(base, first, ref)
    if name == "wrong_ah":
        ref = next(i for i, s in enumerate(prm) if s[3] > 0 and s[1] > 0)
        return _sos_byte(base, ref, "AhAl", ((prm[ref][3] + 1) << 4) | prm[ref][3])
    if name == "ac_before_dc":                         # the DC first scan dropped: the next scan is an AC one
        return _keep_scans(base, lambda i: not (prm[i][1] == 0 and prm[i][3] == 0))
    if name == "two_component_ac":                     # JERR_BAD_PROGRESSION: the reference stops too
        p = mj.params_from_switches(["-revert", "-progressive"], 64, 48, 3)
        jpeg = O.oracle_encode(p, O.synth_image(3, 64, 48)).jpeg
        i = next(k for k, s in enumerate(sos_params(jpeg)) if len(s[0]) > 1)
        _, a, _ = [s for s in segments(jpeg) if s[0] == 0xDA][i]
        off = a + 5 + 2 * jpeg[a + 4]                 # Ss, Se = 1, 5 on a three-component scan
        return jpeg[:off] + bytes([1, 5]) + jpeg[off + 2:]
    if name == "al_14":                                # JERR_BAD_PROGRESSION: Al above 13 in the first (DC) scan
        return _sos_byte(base, 0, "AhAl", 14)
    if name == "two_component_ac_tables":              # JERR_BAD_PROGRESSION: an AC scan of two components, tables defined
        p = mj.params_from_switches(["-revert", "-progressive"], 64, 48, 3)
        jpeg = O.oracle_encode(p, O.synth_image(3, 64, 48)).jpeg
        prm = sos_params(jpeg)
        i = next(k for k, s in enumerate(prm) if s[0] == (1,) and s[1] > 0)
        _, a, _ = [s for s in segments(jpeg) if s[0] == 0xDA][i]
        hl = struct.unpack(">H", jpeg[a + 2:a + 4])[0]
        sel, tail = jpeg[a + 5:a + 7], jpeg[a + 7:a + 10]                  # (Cs, Td/Ta) of component 1; Ss, Se, Ah/Al
        hdr = b"\xff\xda" + struct.pack(">H", 2 + 1 + 4 + 3) + b"\x02" + sel + bytes([jpeg[a + 5] + 1]) + sel[1:] + tail
        return jpeg[:a] + hdr + jpeg[a + 2 + hl:]
    if name == "truncated":
        return base[:len(base) * 2 // 3]
    if name == "corrupt":                              # the first AC scan's data overwritten by 0xFF 0x00 pairs
        i = next(k for k, s in enumerate(prm) if s[1] > 0)
        _, a, b = [s for s in segments(base) if s[0] == 0xDA][i]
        hdr = 2 + struct.unpack(">H", base[a + 2:a + 4])[0]
        n = (b - a - hdr) // 2
        return base[:a + hdr] + b"\xff\x00" * n + base[a + hdr + 2 * n:]
    raise KeyError(name)


def all_sources():
    """(id, bytes) of every source"""
    for c in CASES:
        yield c[0], source(c)
    for name in EXTRA_IDS:
        yield name, extra_source(name)


def md5(b) -> str:
    return hashlib.md5(b if isinstance(b, bytes) else np.ascontiguousarray(b).tobytes()).hexdigest()


def md5_planes(planes) -> str:
    m = hashlib.md5()
    for a in planes:
        m.update(np.ascontiguousarray(a, dtype=np.int16).tobytes())
    return m.hexdigest()


REFSMOOTH = os.path.join(os.path.dirname(GOLD), "..", "build", "librefsmooth.so")
_smooth_lib = None


def ref_smooths(jpeg: bytes):
    """whether the reference library's default decompression block-smooths the file: its pixels with
    do_block_smoothing on differ from those with it off (build/librefsmooth.so); None where it cannot decode it"""
    import ctypes as C
    global _smooth_lib
    if _smooth_lib is None:
        _smooth_lib = C.CDLL(REFSMOOTH)
        _smooth_lib.refsmooth_decompress.argtypes = [C.c_char_p, C.c_ulong, C.c_int, C.c_void_p, C.c_ulong]
        _smooth_lib.refsmooth_decompress.restype = C.c_long
    px = []
    for on in (1, 0):
        buf = C.create_string_buffer(1 << 26)
        n = _smooth_lib.refsmooth_decompress(jpeg, len(jpeg), on, buf, len(buf))
        if n < 0:
            return None
        px.append(buf.raw[:n])
    return px[0] != px[1]


# ----------------------------------------------------------------------------- restatement of the reference's checks
def progression(jpeg: bytes):
    """start_pass_phuff_decoder's checks (jdphuff.c:91-144) over the file's scans: ("ok", coef_bits), ("bad", scan)
    for JERR_BAD_PROGRESSION, ("bogus", scan) for what the reference only warns on (JWRN_BOGUS_PROGRESSION) and for a
    second first scan of a coefficient, which the library refuses as well"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(jpeg)
    if info.sof != 0xC2:
        return "sequential", None
    cb = [[-1] * 64 for _ in range(4)]
    for n, s in enumerate(info.scans):
        dc = s.Ss == 0
        bad = s.Se != 0 if dc else (s.Ss > s.Se or s.Se >= 64 or s.comps_in_scan != 1)
        if (s.Ah != 0 and s.Al != s.Ah - 1) or s.Al > 13:
            bad = True
        if bad:
            return "bad", n
        for i in range(s.comps_in_scan):
            c = cb[s.component_index[i]]
            if not dc and c[0] < 0:
                return "bogus", n
            for k in range(s.Ss, s.Se + 1):
                if s.Ah != max(c[k], 0) or (s.Ah == 0 and c[k] >= 0):
                    return "bogus", n
                c[k] = s.Al
    return "ok", cb


def smoothing_applies(jpeg: bytes) -> bool:
    """smoothing_ok (jdcoefct.c:359-421) after the whole file is read, for a file progression() accepts"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(jpeg)
    verdict, cb = progression(jpeg)
    if verdict == "sequential":
        return False
    assert verdict == "ok"
    useful = False
    for c in range(info.num_components):
        if not info.comp_quant_present[c]:
            return False
        q = info.comp_quant[c]
        if any(q[p] == 0 for p in (0, 1, 8, 16, 9, 2, 3, 10, 17, 24)) or cb[c][0] < 0:
            return False
        useful |= any(cb[c][k] != 0 for k in range(1, 10))
    return useful
