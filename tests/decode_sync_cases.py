"""Sources of the synchronisation tests of the device entropy decode (tests/test_decode_sync.py): generated coefficient
planes written by the repository's CPU oracle, a restatement of where build_decode_batch puts each restart segment's
subsequences, and a serial model of the decode of sequential Huffman files for damaged input.

Entropy coding is lossless, so no golden is needed: a file the oracle writes from planes P decodes to P.  Every
generator is seeded, so a failing case reproduces."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _decode_define(name: str) -> int:
    src = open(os.path.join(ROOT, "mozjpeg_b200", "csrc", "decode.cuh")).read()
    return int(re.search(r"#define\s+%s\s+(\d+)" % name, src).group(1))


DEC_SUB_BITS = _decode_define("DEC_SUB_BITS")      # bits per speculatively decoded subsequence
DEC_CTA = _decode_define("DEC_CTA")                # subsequences per CTA of the synchronisation kernel

# per component (h, v) sampling factors; "cmyk" is a YCCK file with 4:2:0 chroma and full-size K (10 blocks per MCU)
LAYOUTS = {
    "gray": [(1, 1)],
    "1x1": [(1, 1)] * 3,
    "2x1": [(2, 1), (1, 1), (1, 1)],
    "1x2": [(1, 2), (1, 1), (1, 1)],
    "2x2": [(2, 2), (1, 1), (1, 1)],
    "3x2": [(3, 2), (1, 1), (1, 1)],
    "4x1": [(4, 1), (1, 1), (1, 1)],
    "1x4": [(1, 4), (1, 1), (1, 1)],
    "2x2,2x1,1x2": [(2, 2), (2, 1), (1, 2)],
    "2x2,2x2,2x1": [(2, 2), (2, 2), (2, 1)],
    "cmyk": [(2, 2), (1, 1), (1, 1), (2, 2)],
}
# the layouts the pixel routes take (gray, 4:4:4, 4:2:2, 4:4:0, 4:2:0)
PIXEL_LAYOUTS = ("gray", "1x1", "2x1", "1x2", "2x2")


def block_dims(layout, W, H):
    """per component (hib, wib), as jdinput.c initial_setup computes them"""
    f = LAYOUTS[layout]
    hmax, vmax = max(h for h, _ in f), max(v for _, v in f)
    return [(-(-H * v // (vmax * 8)), -(-W * h // (hmax * 8))) for h, v in f]


def _zz():
    from adversarial_cases import ZZ
    return np.asarray(ZZ)


# ------------------------------------------------------------------------------------------------------- contents
def coef_max(precision):
    """largest AC magnitude: size 10 at 8 bits, 14 at 12 bits"""
    return (1 << (precision + 2)) - 1


def planes(content, layout, W, H, precision=8, seed=0):
    """per component a (hib, wib, 64) int16 plane in natural order"""
    import adversarial_cases as AC
    rng = np.random.default_rng(seed)
    dims = block_dims(layout, W, H)
    f = LAYOUTS[layout]
    mx = coef_max(precision)
    zz = _zz()
    out = []
    for c, (hb, wb) in enumerate(dims):
        n = hb * wb
        a = np.zeros((hb, wb, 64), np.int64)
        if content == "zero":
            pass
        elif content == "dc_walk":                    # DC differences through every size, 0 .. precision + 3
            sizes = np.roll(np.arange(precision + 4), c)
            a[..., 0] = AC.dc_walk(sizes, n).reshape(hb, wb)
        elif content == "dense":                      # every coefficient uniform in +-coef_max: blocks past 1024 bits
            a[:] = rng.integers(-mx, mx + 1, (hb, wb, 64))
        elif content == "sparse_zrl":                 # a few values with zero runs of 16 and more between them (ZRL chains)
            a[..., 0] = rng.integers(-40, 41, (hb, wb))
            for y in range(hb):
                for x in range(wb):
                    k = int(rng.integers(1, 8))
                    while k < 64:
                        a[y, x, zz[k]] = int(rng.choice([-1, 1])) * int(rng.integers(1, 1 << int(rng.integers(1, precision + 3))))
                        k += int(rng.integers(17, 40))
        elif content == "periodic":                   # one MCU repeated; every block of the MCU different, none zero
            h, v = f[c]
            y, x = np.meshgrid(np.arange(hb) % v, np.arange(wb) % h, indexing="ij")
            slot = y * h + x
            a[..., 0] = 5 + 7 * c + 3 * slot
            for s in range(h * v):
                for k in range(1, 6):
                    a[slot == s, zz[k + 2 * c + s]] = ((k + c + s) % 5 + 1) * (1 if (k + s) % 2 else -1)
        elif content == "regions":                    # dense top band, sparse middle, zero bottom: very different densities
            t, m = hb // 3, 2 * hb // 3
            a[:t] = rng.integers(-mx, mx + 1, (t, wb, 64))
            a[t:m, :, 0] = rng.integers(-3, 4, (m - t, wb))
            a[t:m, :, zz[1]] = rng.integers(-1, 2, (m - t, wb))
        elif content == "mixed":                      # photo-like: magnitudes falling with the zigzag index
            scale = (mx + 1) / (1 + np.arange(64)) ** 1.5
            v = rng.laplace(0, 1, (hb, wb, 64)) * scale[zz.argsort()] / 8
            a[:] = np.clip(np.round(v), -mx, mx)
            a[..., 0] = np.clip(np.cumsum(rng.integers(-30, 31, n)).reshape(hb, wb), -mx, mx)
        else:
            raise KeyError(content)
        out.append(a.astype(np.int16))
    return out


# ---------------------------------------------------------------------------------------------------- parameters
def _random_script(ncomp, precision, rng, interleave_dc=True):
    """a valid progression: DC Al chains, AC bands cut at random points each with its own Al chain, scans in a random
    order that keeps every chain in order and every AC scan after its component's DC first scan"""
    from mozjpeg_b200 import _abi as A
    max_al = 13 if precision == 12 else 10
    for _ in range(100):
        chains = []
        al = int(rng.integers(0, 4))
        dc_groups = [tuple(range(ncomp))] if interleave_dc else [(c,) for c in range(ncomp)]
        for g in dc_groups:
            chains.append([(g, 0, 0, 0, al)] + [(g, 0, 0, a, a - 1) for a in range(al, 0, -1)])
        for c in range(ncomp):
            cuts = sorted(set(int(x) for x in rng.integers(2, 64, int(rng.integers(0, 3)))))
            edges = [1] + cuts + [64]
            for lo, hi in zip(edges[:-1], edges[1:]):
                al = int(rng.integers(0, 4))
                if rng.random() < 0.15:
                    al = int(rng.integers(4, max_al + 1))
                chains.append([((c,), lo, hi - 1, 0, al)] + [((c,), lo, hi - 1, a, a - 1) for a in range(al, 0, -1)])
        if sum(len(ch) for ch in chains) <= A.MAX_SCANS:
            break
    if precision == 12 and not any(s[4] == 13 for ch in chains for s in ch):
        chains[-1] = [(chains[-1][0][0], chains[-1][0][1], chains[-1][0][2], 0, 13)] + \
                     [(chains[-1][0][0], chains[-1][0][1], chains[-1][0][2], a, a - 1) for a in range(13, 0, -1)]
    script, dc_done = [], set()
    while chains:
        ok = [i for i, ch in enumerate(chains) if ch[0][1] == 0 or ch[0][0][0] in dc_done]
        i = ok[int(rng.integers(0, len(ok)))]
        s = chains[i].pop(0)
        if s[1] == 0 and s[3] == 0:
            dc_done.update(s[0])
        script.append(s)
        if not chains[i]:
            chains.pop(i)
    return script


def params(layout, W, H, precision=8, optimize=False, restart=None, scans="seq", seed=0):
    """b200jpeg_params for the oracle's coefficient encode.  scans: "seq" (one interleaved scan), "multi" (one scan per
    component), "prog" (the standard progressive script), "script" (a seeded random valid script); restart: None,
    "<n>B" (every n MCUs) or "<n>" (every n MCU rows)"""
    import ctypes as C
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    f = LAYOUTS[layout]
    extra = (["-precision", "12"] if precision == 12 else []) + (["-optimize"] if optimize else []) + \
            (["-restart", restart] if restart else [])
    if layout == "cmyk":
        p = mj.params_from_switches(["-revert", *extra], W, H, 3)
        q = mj.tj3_params(W, H, quality=75, subsamp="420", cmyk=True, colorspace=A.CS_YCCK)
        p.num_components, p.jpeg_color_space, p.in_color_space, p.input_components = 4, q.jpeg_color_space, q.in_color_space, 4
        p.write_JFIF_header, p.write_Adobe_marker = q.write_JFIF_header, q.write_Adobe_marker
        p.comp_info[3] = q.comp_info[3]
        p.comp_info[3].quant_tbl_no, p.comp_info[3].dc_tbl_no, p.comp_info[3].ac_tbl_no = 0, 0, 0
    elif layout == "gray":
        p = mj.params_from_switches(["-revert", *extra], W, H, 1)
    else:
        p = mj.params_from_switches(["-revert", "-sample", layout, *extra], W, H, 3)
    for c, (h, v) in enumerate(f):
        p.comp_info[c].h_samp_factor, p.comp_info[c].v_samp_factor = h, v
    nc = p.num_components
    if scans == "multi":
        p.num_scans = nc
        for k in range(nc):
            s = p.scan_info[k]
            s.comps_in_scan, s.Ss, s.Se, s.Ah, s.Al = 1, 0, 63, 0, 0
            s.component_index[0] = k
    elif scans == "prog":
        A.check(A.load().b200jpeg_simple_progression(C.byref(p)), "simple_progression")
    elif scans == "script":
        blocks = sum(h * v for h, v in f)
        script = _random_script(nc, precision, np.random.default_rng(seed), interleave_dc=blocks <= 10)
        p.num_scans = len(script)
        for k, (comps, ss, se, ah, al) in enumerate(script):
            s = p.scan_info[k]
            s.comps_in_scan, s.Ss, s.Se, s.Ah, s.Al = len(comps), ss, se, ah, al
            for i, c in enumerate(comps):
                s.component_index[i] = c
    else:
        assert scans == "seq"
    if scans in ("prog", "script"):
        p.optimize_scans = 0
    return p


def encode(planes_, layout, W, H, **kw) -> bytes:
    from oracle import oracle as O
    return O.oracle_encode_coefs(params(layout, W, H, **kw), planes_)


# (id, layout, width, height, content, precision, optimize, restart, scans, seed): ragged sizes, so interleaved scans carry
# dummy blocks; every layout, content, table choice, precision, restart kind and scan kind appears, not their product
CASES = [
    ("gray_zero", "gray", 61, 37, "zero", 8, False, None, "seq", 1),
    ("gray_dc_walk", "gray", 203, 45, "dc_walk", 8, False, None, "seq", 2),
    ("gray_dc_walk12", "gray", 203, 45, "dc_walk", 12, True, "1B", "seq", 3),
    ("gray_dense", "gray", 93, 70, "dense", 8, False, None, "seq", 4),
    ("gray_dense12", "gray", 93, 70, "dense", 12, True, None, "seq", 5),
    ("gray_sparse_zrl", "gray", 130, 61, "sparse_zrl", 8, False, "7B", "seq", 6),
    ("444_periodic", "1x1", 61, 37, "periodic", 8, False, None, "seq", 7),
    ("444_dense_restart_rows", "1x1", 77, 53, "dense", 8, True, "1", "seq", 8),
    ("422_regions", "2x1", 181, 99, "regions", 8, False, "5B", "seq", 9),
    ("440_mixed_opt", "1x2", 99, 181, "mixed", 8, True, None, "seq", 10),
    ("420_periodic", "2x2", 61, 37, "periodic", 8, False, None, "seq", 11),
    ("420_dense", "2x2", 77, 53, "dense", 8, False, "1B", "seq", 12),
    ("420_mixed_multi", "2x2", 133, 75, "mixed", 8, True, "3B", "multi", 13),
    ("3x2_periodic", "3x2", 61, 37, "periodic", 8, False, None, "seq", 14),
    ("3x2_dense12", "3x2", 61, 37, "dense", 12, True, "7B", "seq", 15),
    ("4x1_periodic", "4x1", 61, 37, "periodic", 8, False, "1", "seq", 16),
    ("4x1_sparse_multi", "4x1", 75, 41, "sparse_zrl", 8, True, None, "multi", 17),
    ("1x4_periodic", "1x4", 61, 37, "periodic", 8, False, None, "seq", 18),
    ("1x4_regions12", "1x4", 61, 77, "regions", 12, True, "1B", "seq", 19),
    ("221_periodic", "2x2,2x1,1x2", 61, 37, "periodic", 8, False, None, "seq", 20),
    ("221_dense", "2x2,2x1,1x2", 61, 37, "dense", 8, True, "2B", "seq", 21),
    ("222_periodic", "2x2,2x2,2x1", 61, 37, "periodic", 8, False, "1", "seq", 22),
    ("222_mixed_multi", "2x2,2x2,2x1", 61, 37, "mixed", 8, False, "7B", "multi", 23),
    ("cmyk_periodic", "cmyk", 61, 37, "periodic", 8, False, None, "seq", 24),
    ("cmyk_dense12", "cmyk", 45, 29, "dense", 12, True, "1B", "seq", 25),
    # progressive: the standard script, and seeded valid scripts
    ("prog_420_mixed", "2x2", 133, 75, "mixed", 8, False, None, "prog", 26),
    ("prog_gray_dense_restart", "gray", 93, 70, "dense", 8, False, "1B", "prog", 27),
    ("prog_221_periodic", "2x2,2x1,1x2", 61, 37, "periodic", 8, False, "7B", "prog", 28),
    ("prog_cmyk_mixed", "cmyk", 61, 37, "mixed", 8, False, "1", "prog", 29),
    ("prog12_3x2_mixed", "3x2", 61, 37, "mixed", 12, False, None, "prog", 30),
    ("script_gray_mixed", "gray", 93, 70, "mixed", 8, False, None, "script", 31),
    ("script_444_dense", "1x1", 61, 37, "dense", 8, False, "3B", "script", 32),
    ("script_420_regions", "2x2", 133, 75, "regions", 8, False, None, "script", 33),
    ("script_4x1_sparse", "4x1", 75, 41, "sparse_zrl", 8, False, "1", "script", 34),
    ("script12_gray_dense", "gray", 61, 37, "dense", 12, False, "7B", "script", 35),
    ("script12_1x4_mixed", "1x4", 61, 77, "mixed", 12, False, None, "script", 36),
    ("script_cmyk_periodic", "cmyk", 45, 29, "periodic", 8, False, None, "script", 37),
    ("script_222_dc_walk", "2x2,2x2,2x1", 61, 37, "dc_walk", 8, False, "2B", "script", 38),
]
CASE = {c[0]: c for c in CASES}

# the coefficient families of tests/adversarial_cases.py, written sequential (standard and optimal tables) and progressive
FAMILY_CASES = [(f"family_{fam}_{prec}_{kind}", fam, prec, kind) for prec in (8, 12)
                for fam in ("fib", "fib_dc", "equal", "single_symbol", "all_symbols", "max_magnitude")
                for kind in (("seq", "seq_opt", "prog") if prec == 8 else ("seq", "prog"))]   # 12-bit files get optimal tables


def case_source(cid):
    """(file, planes, params keywords, layout) of a CASES or FAMILY_CASES id"""
    if cid.startswith("family_"):
        import adversarial_cases as AC
        fam, prec, kind = next((f, p, k) for i, f, p, k in FAMILY_CASES if i == cid)
        pl = AC.coef_families(prec)[fam]
        hb, wb = pl[0].shape[:2]
        kw = dict(precision=prec, optimize=kind == "seq_opt", scans="prog" if kind == "prog" else "seq")
        return encode(pl, "gray", wb * 8, hb * 8, **kw), pl, kw, "gray", wb * 8, hb * 8
    _, layout, W, H, content, prec, opt, rst, scans, seed = CASE[cid]
    pl = planes(content, layout, W, H, prec, seed)
    kw = dict(precision=prec, optimize=opt, restart=rst, scans=scans, seed=seed)
    return encode(pl, layout, W, H, **kw), pl, kw, layout, W, H


# ------------------------------------------------------------------------------------------------ segment placement
def scan_data_end(d: bytes, pos: int) -> int:
    """the end of the entropy-coded data from pos: the first 0xFF that starts a marker other than RSTn; FF FF 00 ends
    it too (source.cpp scan_data_end)"""
    n = len(d)
    while pos < n:
        q = d.find(b"\xff", pos)
        if q < 0:
            return n
        r = q + 1
        while r < n and d[r] == 0xFF:
            r += 1
        if r >= n:
            return q
        if (d[r] == 0 and r == q + 1) or 0xD0 <= d[r] <= 0xD7:
            pos = r + 1
            continue
        return q
    return n


class Refused(Exception):
    """the device decode refuses the file (the words say why)"""


def unstuff(d: bytes, lo: int, end: int, ri: int, nseg: int):
    """the unstuffed bytes of each restart segment of the scan data d[lo:end] (build_decode_batch): fill bytes dropped,
    FF 00 taken as FF, RSTn checked against the segment number; refused where the scan ends early"""
    segs, p = [], lo
    for sg in range(nseg):
        out, rst = bytearray(), False
        while p < end:
            q = d.find(b"\xff", p, end)
            q = end if q < 0 else q
            out += d[p:q]
            p = q
            if p >= end:
                break
            r = p + 1
            while r < end and d[r] == 0xFF:
                r += 1
            if r >= end:
                p = end
                break
            if d[r] == 0:
                out.append(0xFF)
                p = r + 1
                continue
            if not ri:
                raise Refused("restart marker in a scan without restart interval")
            if d[r] - 0xD0 != sg & 7:
                raise Refused(f"restart marker RST{d[r] - 0xD0} where RST{sg & 7} was due")
            p, rst = r + 1, True
            break
        if not rst and p >= end and sg + 1 < nseg:
            raise Refused(f"scan ends after {sg + 1} of its {nseg} restart segments")
        segs.append(bytes(out))
    return segs


def _geometry(info):
    nc = info.num_components
    hmax = max(info.h_samp_factor[c] for c in range(nc))
    vmax = max(info.v_samp_factor[c] for c in range(nc))
    W, H = info.image_width, info.image_height
    wib = [-(-W * info.h_samp_factor[c] // (hmax * 8)) for c in range(nc)]
    hib = [-(-H * info.v_samp_factor[c] // (vmax * 8)) for c in range(nc)]
    return hmax, vmax, wib, hib


def scan_layout(info, sc):
    """(MCUs, MCUs per row, [(component, dx, dy)] per MCU slot) of a scan (build_decode_batch)"""
    hmax, vmax, wib, hib = _geometry(info)
    comps = [sc.component_index[i] for i in range(sc.comps_in_scan)]
    if len(comps) == 1:
        c = comps[0]
        return wib[c] * hib[c], wib[c], [(c, 0, 0)]
    per_row = -(-info.image_width // (hmax * 8))
    mcus = per_row * -(-info.image_height // (vmax * 8))
    slots = [(c, x, y) for c in comps for y in range(info.v_samp_factor[c]) for x in range(info.h_samp_factor[c])]
    return mcus, per_row, slots


def _is_first_scan(info, sc):
    return info.sof != 0xC2 or sc.Ah == 0


def segment_table(files):
    """per restart segment of the speculative decode, in build_decode_batch's order (image, scan, restart segment;
    refinement scans have no subsequences): dict(img, scan, seg, nbytes, sub0, nsub, nmcu)"""
    from mozjpeg_b200 import jpegtran as T
    out, sub = [], 0
    for i, f in enumerate(files):
        info = T.parse_source(f)
        for k in range(info.num_scans):
            sc = info.scans[k]
            mcus, _, _ = scan_layout(info, sc)
            ri = sc.restart_interval
            nseg = -(-mcus // ri) if ri else 1
            segs = unstuff(f, sc.data_offset, sc.data_offset + sc.data_size, ri, nseg)
            if not _is_first_scan(info, sc):
                continue
            for sg, b in enumerate(segs):
                nsub = max(1, -(-8 * len(b) // DEC_SUB_BITS))
                nmcu = min(ri, mcus - sg * ri) if ri else mcus
                out.append(dict(img=i, scan=k, seg=sg, nbytes=len(b), sub0=sub, nsub=nsub, nmcu=nmcu))
                sub += nsub
    return out


def total_subsequences(files) -> int:
    t = segment_table(files)
    return t[-1]["sub0"] + t[-1]["nsub"] if t else 0


# ------------------------------------------------------------------------------------------------- the serial model
def _codes(h):
    """{(length, code): symbol} of a b200jpeg_huff_tbl"""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(h.bits[ln]):
            out[(ln, code)] = h.huffval[k]
            code += 1
            k += 1
        code <<= 1
    return out


def _extend(x, s):
    return x - (1 << s) + 1 if s and x < (1 << (s - 1)) else x


def _s16(v):
    return ((v + 32768) & 0xFFFF) - 32768


def serial_decode(jpeg: bytes, info=None, block_starts=None):
    """The planes the device decode makes of a sequential Huffman file, or Refused.  A plain restatement of
    build_decode_batch's unstuffing and of decode_mcu (jdhuff.c:564-647) with the device's semantics: an invalid code,
    a symbol that needs bits past its segment's end, a wrong RSTn, a scan that ends early and FF FF 00 inside the data
    are refused; fill bytes in front of a marker are skipped, an AC run past 63 writes position 63, and whatever follows
    a segment's last MCU is ignored.  info: the parsed headers (those of the undamaged file for a damaged one, whose
    headers are the same); the data end is found here.  block_starts: a list that receives, per segment of the
    speculative decode, the bit offsets at which its blocks start."""
    from mozjpeg_b200 import jpegtran as T
    if info is None:
        info = T.parse_source(jpeg)
    if info.sof not in (0xC0, 0xC1):
        raise ValueError("sequential files only")
    hmax, vmax, wib, hib = _geometry(info)
    nc = info.num_components
    out = [np.zeros((hib[c], wib[c], 64), np.int16) for c in range(nc)]
    zz = _zz()
    for k in range(info.num_scans):
        sc = info.scans[k]
        lo = sc.data_offset
        end = scan_data_end(jpeg, lo)
        r = end
        while r < len(jpeg) and jpeg[r] == 0xFF:
            r += 1
        if r < len(jpeg) and jpeg[r] == 0 and r > end:
            raise Refused("0xFF 0x00 where a marker is due")
        mcus, per_row, slots = scan_layout(info, sc)
        ri = sc.restart_interval
        nseg = -(-mcus // ri) if ri else 1
        segs = unstuff(jpeg, lo, end, ri, nseg)
        comps = [sc.component_index[i] for i in range(sc.comps_in_scan)]
        dct = {c: _codes(info.huff[sc.dc_huff[i]]) for i, c in enumerate(comps)}
        act = {c: _codes(info.huff[sc.ac_huff[i]]) for i, c in enumerate(comps)}
        mx = {c: (1 if len(comps) == 1 else info.h_samp_factor[c]) for c in comps}
        my = {c: (1 if len(comps) == 1 else info.v_samp_factor[c]) for c in comps}
        for sg, data in enumerate(segs):
            nbits = 8 * len(data)
            bits = int.from_bytes(data, "big") << 32                 # zero bits behind the data, as in the word buffer
            total = nbits + 32
            pos = 0

            def symbol(table):
                nonlocal pos
                code = 0
                for ln in range(1, 17):
                    code = (code << 1) | ((bits >> (total - 1 - pos - ln + 1)) & 1)
                    sym = table.get((ln, code))
                    if sym is not None:
                        return ln, sym
                raise Refused("invalid Huffman code")

            def take(ln, n):
                nonlocal pos
                if pos + ln + n > nbits:
                    raise Refused("too few bits for the segment's MCUs")
                x = (bits >> (total - pos - ln - n)) & ((1 << n) - 1) if n else 0
                pos += ln + n
                return x

            starts = []
            nmcu = min(ri, mcus - sg * ri) if ri else mcus
            pred = {c: 0 for c in comps}
            for m in range(sg * ri if ri else 0, (sg * ri if ri else 0) + nmcu):
                for c, dx, dy in slots:
                    starts.append(pos)
                    col, row = (m % per_row) * mx[c] + dx, (m // per_row) * my[c] + dy
                    blk = out[c][row, col] if col < wib[c] and row < hib[c] else np.zeros(64, np.int16)
                    ln, s = symbol(dct[c])
                    pred[c] += _extend(take(ln, s), s)
                    blk[0] = _s16(pred[c])
                    kk = 1
                    while kk < 64:
                        ln, sym = symbol(act[c])
                        rr, s = sym >> 4, sym & 15
                        x = take(ln, s)
                        if s:
                            kk += rr
                            blk[zz[min(kk, 63)]] = _extend(x, s)
                            kk += 1
                        elif rr == 15:
                            kk += 16
                        else:
                            break
            if block_starts is not None:
                block_starts.append(starts)
    return out


# --------------------------------------------------------------------------------------------------------- damage
_MARKER = re.compile(rb"\xff+([^\x00\xff])")


def _marker_kinds(d: bytes, lo: int):
    """the markers from lo on, RSTn counted as one kind"""
    return [b"R" if 0xD0 <= m.group(1)[0] <= 0xD7 else m.group(1) for m in _MARKER.finditer(d, lo)]


MUTANT_SOURCES = [                                  # (id, layout, width, height, precision, restart)
    ("gray16", "gray", 16, 16, 8, None),
    ("gray40_rst", "gray", 40, 24, 8, "1B"),
    ("420_48", "2x2", 48, 32, 8, None),
    ("420_64_rst", "2x2", 64, 48, 8, "1B"),
    ("422_40", "2x1", 40, 24, 8, None),
    ("422_56_rst", "2x1", 56, 40, 8, "2B"),
    ("gray12_32", "gray", 32, 24, 12, None),
    ("gray12_48_rst", "gray", 48, 32, 12, "1"),
]


def mutant_source(sid):
    """a small sequential file with restart markers where asked, and its planes (mixed content, standard tables at 8
    bits: some stuffed bytes)"""
    _, layout, W, H, prec, rst = next(m for m in MUTANT_SOURCES if m[0] == sid)
    pl = planes("mixed", layout, W, H, prec, seed=W * H + prec)
    return encode(pl, layout, W, H, precision=prec, optimize=prec == 12, restart=rst), pl


def mutants(good: bytes, n: int, seed: int):
    """n seeded damaged copies of a one-scan file: single bit flips, byte deletions and insertions inside the
    entropy-coded data, RSTn renumbering and truncations (the data cut and EOI appended).  A mutant that creates or
    removes a marker inside the data (other than by truncation, and RSTn renumbering aside) is dropped, so that model
    and device see the same marker structure.  [(kind, bytes)]"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(good)
    sc = info.scans[0]
    lo, hi = sc.data_offset, sc.data_offset + sc.data_size
    want = _marker_kinds(good, lo)
    rsts = [m.start(1) for m in re.finditer(rb"\xff([\xd0-\xd7])", good[lo:hi])]
    rng = np.random.default_rng(seed)
    kinds = ["flip", "flip", "flip", "delete", "insert", "truncate"] + (["renumber"] if rsts else [])
    out, tries = [], 0
    while len(out) < n and tries < 50 * n:
        tries += 1
        kind = kinds[int(rng.integers(0, len(kinds)))]
        d = bytearray(good)
        if kind == "flip":
            p = int(rng.integers(lo, hi))
            d[p] ^= 1 << int(rng.integers(0, 8))
        elif kind == "delete":
            del d[int(rng.integers(lo, hi))]
        elif kind == "insert":
            d.insert(int(rng.integers(lo, hi + 1)), int(rng.integers(0, 256)))
        elif kind == "renumber":
            p = lo + rsts[int(rng.integers(0, len(rsts)))]
            d[p] = 0xD0 + (d[p] - 0xD0 + int(rng.integers(1, 8))) % 8
        else:
            d = d[:int(rng.integers(lo, hi))] + bytearray(b"\xff\xd9")
        d = bytes(d)
        if kind != "truncate" and _marker_kinds(d, lo) != want:
            continue
        out.append((kind, d))
    return out


def model(jpeg: bytes, info):
    """serial_decode's planes, or None where it refuses"""
    try:
        return serial_decode(jpeg, info)
    except Refused:
        return None


# ------------------------------------------------------------------------------------------------- placed boundaries
# Gray files with the standard tables and nothing but DC values: a block whose DC difference is 0 costs 6 bits (DC size
# 0, EOB), one whose difference is +-1 costs 8 (DC size 1 and its bit, EOB), so segment lengths can be dialled exactly.
def dc_segment(R, d):
    """R DC values whose differences from a predictor of 0 are nonzero exactly d times (the first d blocks): 6R + 2d bits"""
    if d % 2 == 0:
        v = [1, 0] * (d // 2) + [0] * (R - d)
    else:
        v = [1, 0] * (d // 2) + [1] * (R - d + 1)
    return np.asarray(v[:R], np.int16)


def dc_file(wib, hib, dcs, restart=None):
    """a gray (hib * 8, wib * 8) file of the given DC values (raster order) and its planes"""
    pl = np.zeros((hib, wib, 64), np.int16)
    pl[..., 0] = np.asarray(dcs, np.int16).reshape(hib, wib)
    return encode([pl], "gray", wib * 8, hib * 8, restart=restart), [pl]


def spacer_counts(wib, hib):
    """{restart (None or "<n>B"): subsequences} of all-zero gray spacer files of one geometry"""
    out = {}
    n = wib * hib
    for R in [None] + [r for r in list(range(1, 17)) + [20, 24, 32, 48, 64, 96, 128, 170, 256, 512] if r <= n]:
        f, _ = dc_file(wib, hib, np.zeros(n), None if R is None else f"{R}B")
        out.setdefault(total_subsequences([f]), None if R is None else f"{R}B")
    return {v: k for k, v in out.items()}


def spacers_for(offset, wib, hib):
    """all-zero gray files of the geometry whose subsequences add up to offset modulo DEC_CTA (fewest files)"""
    counts = spacer_counts(wib, hib)
    best = {0: []}
    for _ in range(8):
        nxt = dict(best)
        for r, files in best.items():
            for rst, cnt in counts.items():
                t = (r + cnt) % DEC_CTA
                if t not in nxt or len(nxt[t]) > len(files) + 1:
                    nxt[t] = files + [rst]
        best = nxt
        if offset % DEC_CTA in best:
            break
    n = wib * hib
    return [dc_file(wib, hib, np.zeros(n), rst) for rst in best[offset % DEC_CTA]]


def _lengths_case(R, targets):
    """one gray file, restart every R blocks (one block row per segment), segment k dialled to targets[k] bytes"""
    dcs = []
    for L in targets:
        d = 4 * L - 3 * R
        assert 0 <= d <= R, (R, L)
        dcs.append(dc_segment(R, d))
    return dc_file(R, len(targets), np.concatenate(dcs), f"{R}B")


# (seed, blocks across, blocks down) of eobrun_file for the two EOB-run placements (found by search; placed() asserts them)
EOBRUN_SEEDS = {"eobrun_at_subsequence_end": (7, 64, 48), "eobrun_across_cta": (1, 320, 256)}

# id -> what the case places (see placed())
PLACED = ["lengths_128", "lengths_256", "block_on_start", "offset_0", "offset_1", "offset_127", "offset_64",
          "exactly_128", "exactly_128_mid_cta", "periodic_420", "eobrun_at_subsequence_end", "eobrun_across_cta",
          "over_1024_tiles", "restart_129600"]
LARGE = ("over_1024_tiles", "restart_129600")


def placed(pid):
    """(files, planes per file, target index) of a placed case, with its placement asserted through segment_table;
    target: the file whose first segment is placed"""
    if pid in ("lengths_128", "lengths_256"):
        m = 1 if pid == "lengths_128" else 2
        targets = [128 * m, 128 * m - 1, 128 * m + 1, 128 * m + 4]
        f, pl = _lengths_case(160 if m == 1 else 300, targets)
        assert [s["nbytes"] for s in segment_table([f])] == targets
        return [f], [pl], 0
    if pid == "block_on_start":
        # DEC_SUB_BITS / 8 blocks of 8 bits, then 6-bit blocks: a block starts exactly on the second subsequence's start
        f, pl = dc_file(400, 1, dc_segment(400, DEC_SUB_BITS // 8))
        starts = []
        serial_decode(f, block_starts=starts)
        assert DEC_SUB_BITS in starts[0] and segment_table([f])[0]["nsub"] > 2, starts[0][:8]
        return [f], [pl], 0
    if pid.startswith("offset_"):
        off = int(pid.split("_")[1])
        W, H = 256, 128
        pt = planes("dense", "gray", W, H, 8, 7 + off)
        tgt = encode(pt, "gray", W, H)
        sp = spacers_for(off, W // 8, H // 8)
        files = [f for f, _ in sp] + [tgt]
        t = segment_table(files)
        first = next(s for s in t if s["img"] == len(sp))
        assert first["sub0"] % DEC_CTA == off % DEC_CTA and first["nsub"] > 2 * DEC_CTA, first
        return files, [p for _, p in sp] + [pt], len(sp)
    if pid.startswith("exactly_128"):
        n = DEC_SUB_BITS * DEC_CTA // 8                  # blocks of 8 bits that fill DEC_CTA subsequences exactly
        wib = 128
        f, pl = dc_file(wib, n // wib, dc_segment(n, n))
        files, pls = [f], [pl]
        if pid.endswith("mid_cta"):
            sp = spacers_for(DEC_CTA // 2, wib, n // wib)
            files, pls = [g for g, _ in sp] + files, [p for _, p in sp] + pls
        t = segment_table(files)
        s = next(s for s in t if s["img"] == len(files) - 1)
        assert s["nsub"] == DEC_CTA and s["nbytes"] * 8 == DEC_SUB_BITS * DEC_CTA, s
        assert s["sub0"] % DEC_CTA == (DEC_CTA // 2 if pid.endswith("mid_cta") else 0)
        return files, pls, len(files) - 1
    if pid == "periodic_420":                            # one MCU repeated, no restarts: the slowest self-synchronisation
        pl = planes("periodic", "2x2", 1024, 768, 8, 0)
        f = encode(pl, "2x2", 1024, 768)
        assert segment_table([f])[0]["nsub"] >= 2 * DEC_CTA
        return [f], [pl], 0
    if pid.startswith("eobrun_"):
        # seeds found by search: in the AC first scan (scan 1) an EOBr symbol of more than one block ends exactly at a
        # subsequence end, or is the last symbol to start in a CTA's last subsequence, so that the blocks it ends are
        # counted there while the next block starts in the next CTA
        seed, wib, hib = EOBRUN_SEEDS[pid]
        f, pl = eobrun_file(seed, wib, hib)
        seg = next(s for s in segment_table([f]) if s["scan"] == 1)
        syms = ac_first_symbols(f, 1)
        if pid == "eobrun_at_subsequence_end":
            assert any(d > 1 and e % DEC_SUB_BITS == 0 and e < 8 * seg["nbytes"] for _, e, d in syms), seed
        else:
            def crossing(i):
                a, _, d = syms[i]
                j = seg["sub0"] + a // DEC_SUB_BITS
                return d > 1 and j % DEC_CTA == DEC_CTA - 1 and i + 1 < len(syms) and \
                    (seg["sub0"] + syms[i + 1][0] // DEC_SUB_BITS) // DEC_CTA == j // DEC_CTA + 1
            assert any(crossing(i) for i in range(len(syms))), seed
        return [f], [pl], 0
    if pid == "over_1024_tiles":                         # three 4K 4:4:4 files of uniform +-1023: the scan's carry runs
        pl = planes("dense", "1x1", 3840, 2160, 8, 11)
        f = encode(pl, "1x1", 3840, 2160)
        files = [f, f, f]
        assert total_subsequences(files) > 1024 * 1024
        return files, [pl] * 3, 0
    if pid == "restart_129600":                          # a 4K gray frame with a restart marker after every block
        pl = planes("mixed", "gray", 3840, 2160, 8, 12)
        f = encode(pl, "gray", 3840, 2160, restart="1B")
        assert len(segment_table([f])) == 480 * 270
        return [f], [pl], 0
    raise KeyError(pid)


# ------------------------------------------------------------------------------------------- EOB runs of AC first scans
def eobrun_file(seed, wib=64, hib=48):
    """A gray progressive file of two scans (DC first, AC first 1..63, both Al 0, no restarts) whose blocks come in
    groups: one block with a few AC values, then a run of blocks with none, which the AC scan codes as one EOBr symbol"""
    import ctypes as C
    from mozjpeg_b200 import _abi as A
    rng = np.random.default_rng(seed)
    zz = _zz()
    pl = np.zeros((hib * wib, 64), np.int16)
    pl[:, 0] = rng.integers(-20, 21, hib * wib)
    b = 0
    while b < hib * wib:
        for k in sorted(rng.choice(np.arange(1, 64), int(rng.integers(1, 7)), replace=False)):
            pl[b, zz[k]] = int(rng.choice([-1, 1])) * int(rng.integers(1, 1 << int(rng.integers(1, 9))))
        b += 1 + int(rng.integers(1, 40))
    pl = [pl.reshape(hib, wib, 64)]
    p = params("gray", wib * 8, hib * 8, scans="prog")
    p.num_scans = 2
    for k, (ss, se) in enumerate(((0, 0), (1, 63))):
        s = p.scan_info[k]
        s.comps_in_scan, s.Ss, s.Se, s.Ah, s.Al = 1, ss, se, 0, 0
        s.component_index[0] = 0
    from oracle import oracle as O
    return O.oracle_encode_coefs(p, pl), pl


def ac_first_symbols(jpeg: bytes, k: int):
    """[(start bit, end bit, blocks the symbol ends)] of every symbol of scan k, a one-segment AC first scan of a gray
    file (decode_mcu_AC_first, jdphuff.c): an EOBr symbol ends 2^r + its appended bits blocks, any other symbol at
    most one"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(jpeg)
    sc = info.scans[k]
    assert info.num_components == 1 and sc.Ss > 0 and sc.Ah == 0 and not sc.restart_interval
    data = unstuff(jpeg, sc.data_offset, sc.data_offset + sc.data_size, 0, 1)[0]
    nbits = 8 * len(data)
    bits = int.from_bytes(data, "big") << 32
    total = nbits + 32
    table = _codes(info.huff[sc.ac_huff[0]])
    nblocks = -(-info.image_width // 8) * -(-info.image_height // 8)
    out, pos, blk, kk = [], 0, 0, sc.Ss
    while blk < nblocks:
        start, code = pos, 0
        for ln in range(1, 17):
            code = (code << 1) | ((bits >> (total - 1 - pos - ln + 1)) & 1)
            if (ln, code) in table:
                break
        sym = table[(ln, code)]
        r, s = sym >> 4, sym & 15
        n = r if (s == 0 and r != 15) else s
        x = (bits >> (total - pos - ln - n)) & ((1 << n) - 1) if n else 0
        pos += ln + n
        done = 0
        if s:
            kk += r + 1
        elif r == 15:
            kk += 16
        else:
            done, kk = (1 << r) + x, sc.Ss
        if kk > sc.Se:
            done, kk = 1, sc.Ss
        out.append((start, pos, done))
        blk += done
    return out


def wrong_cta_guesses(files):
    """How many subsequences that open a CTA inside a segment of several subsequences start from a wrong guess: the
    speculative decode guesses a block start in MCU slot 0 there, which k_dec_fix must redo unless a block of slot 0
    does start at that bit.  Sequential gray files only (every block is in slot 0), through the serial model."""
    wrong = 0
    table = segment_table(files)
    k = 0
    for f in files:
        starts = []
        serial_decode(f, block_starts=starts)
        for st in starts:
            s = table[k]
            k += 1
            first = -(-s["sub0"] // DEC_CTA) * DEC_CTA
            if s["sub0"] % DEC_CTA == 0:
                first += DEC_CTA
            st = set(st)
            wrong += sum((j - s["sub0"]) * DEC_SUB_BITS not in st for j in range(first, s["sub0"] + s["nsub"], DEC_CTA))
    assert k == len(table)
    return wrong
