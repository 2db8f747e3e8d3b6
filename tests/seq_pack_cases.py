"""Sources of the sequential scan packer's boundary tests (tests/test_seq_pack_boundaries.py): a serial model of the
packed layout k_block_bits_seq / k_scan_layout / k_encode_seq write, placed coefficient planes whose block lengths are
dialled bit for bit under the standard tables, and pixel families whose final planes reach the same rules through the
trellis walks.

The model takes a sequential file's headers (its SOF, DHT, DRI and SOS, through parse_source) and the final quantized
planes, and gives per scan, in the device's block order t: each block's bit string as encode_one_block (jchuff.c:563-661)
writes it, its tile (t // 256), its bit offset with restart padding and marker bits (k_scan_layout's seg_corr), its class
as k_encode_seq decides it (a slot block of at most 128 bits that ends no restart segment, else a fallback block; no
slots at 12 bits), the words it builds with a plain store or an OR, and the stuffed scan bytes.  classes() names the
boundary classes a case reaches; locate() maps a scan byte to its block, tile, word and class.

Every generator is seeded or constructed, so a failing case reproduces."""
import bisect
import functools

import numpy as np

TILE = 256                                  # blocks per CTA of k_block_bits_seq / k_encode_seq
SLOT_BITS = 128                             # SEQ_SLOT_WORDS * 32
ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
               21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
               61, 54, 47, 55, 62, 63])        # zigzag position -> natural index


# ------------------------------------------------------------------------------------------------------ the model
def code_table(h):
    """{symbol: (code, length)} of a b200jpeg_huff_tbl (jchuff.c jpeg_make_c_derived_tbl)"""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(h.bits[ln]):
            out[h.huffval[k]] = (code, ln)
            code += 1
            k += 1
        code <<= 1
    return out


def _nbits(v):
    return int(abs(int(v))).bit_length()


def block_bits(blk, last_dc, dct, act):
    """the bit string ('0'/'1') of one block in natural order under encode_one_block (jchuff.c:563-661)"""
    out = []

    def put(sym, table, v, nb):
        code, ln = table[sym]
        out.append(format(code, "0%db" % ln))
        if nb:
            out.append(format(v & ((1 << nb) - 1), "0%db" % nb))

    d = int(blk[0]) - last_dc
    nb = _nbits(d)
    put(nb, dct, d - 1 if d < 0 else d, nb)
    r = 0
    for k in range(1, 64):
        v = int(blk[ZZ[k]])
        if v == 0:
            r += 1
            continue
        while r > 15:
            put(0xF0, act, 0, 0)
            r -= 16
        nb = _nbits(v)
        put((r << 4) + nb, act, v - 1 if v < 0 else v, nb)
        r = 0
    if r:
        put(0x00, act, 0, 0)
    return "".join(out)


class Block:
    __slots__ = ("t", "comp", "row", "col", "bits", "off", "tile", "j", "seg_end", "pad", "kind", "reason", "words")

    def __repr__(self):
        return "block %d (component %d, block row %d col %d): tile %d index %d, bits %d..%d (%d bits), %s block%s" % (
            self.t, self.comp, self.row, self.col, self.tile, self.j, self.off, self.off + len(self.bits), len(self.bits),
            self.kind, " (%s)" % self.reason if self.reason else "")


class ScanModel:
    """One sequential scan as the device lays it out: blocks (in order t), the unstuffed bit string, the stuffed bytes
    and, per stuffed byte, the unstuffed byte it came from."""

    def __init__(self, k, precision, blocks, seglen, stream, markers, data, src):
        self.k, self.precision, self.blocks, self.seglen = k, precision, blocks, seglen
        self.stream, self.markers, self.data, self.src = stream, markers, data, src
        self.starts = [b.off for b in blocks]
        self.ntiles = -(-len(blocks) // TILE)

    def tile_blocks(self, i):
        return self.blocks[i * TILE:(i + 1) * TILE]

    def block_at(self, bit):
        """the block whose bits, padding or marker hold unstuffed bit `bit`"""
        return self.blocks[max(0, bisect.bisect_right(self.starts, bit) - 1)]

    def locate(self, byte_offset):
        """a scan byte (stuffed, from the scan's first data byte) as block, tile, word and class"""
        if byte_offset >= len(self.data):
            return "scan %d byte %d: past the model's %d bytes" % (self.k, byte_offset, len(self.data))
        u = self.src[byte_offset]
        bit = 8 * u
        b = self.block_at(bit)
        where = "marker or padding after " if bit >= b.off + len(b.bits) else ""
        w = bit >> 5
        built = [x for x in self.blocks[max(0, b.t - 64):b.t + 64] if any(ww == w for ww, _ in x.words)]
        how = ", ".join("%s by block %d" % (s, x.t) for x in built for ww, s in x.words if ww == w)
        inside = ", ".join("%d (%s, %d bits)" % (x.t, x.kind, len(x.bits)) for x in self.blocks[max(0, b.t - 64):b.t + 64]
                           if x.off < 32 * w + 32 and x.off + len(x.bits) > 32 * w)
        return "scan %d byte %d (unstuffed byte %d, word %d: %s; blocks in the word: %s): %s%r" % (
            self.k, byte_offset, u, w, how or "no writer", inside, where, b)


def _scan_slots(info, sc, geom):
    """(MCUs, MCUs per row, [(component, dx, dy)] per MCU slot) of a scan"""
    hmax, vmax, wib, hib = geom
    comps = [sc.component_index[i] for i in range(sc.comps_in_scan)]
    if len(comps) == 1:
        c = comps[0]
        return wib[c] * hib[c], wib[c], [(c, 0, 0)], True
    per_row = -(-info.image_width // (hmax * 8))
    mcus = per_row * -(-info.image_height // (vmax * 8))
    return mcus, per_row, [(c, x, y) for c in comps for y in range(info.v_samp_factor[c]) for x in range(info.h_samp_factor[c])], False


def _geometry(info):
    nc = info.num_components
    hmax = max(info.h_samp_factor[c] for c in range(nc))
    vmax = max(info.v_samp_factor[c] for c in range(nc))
    W, H = info.image_width, info.image_height
    return hmax, vmax, [-(-W * info.h_samp_factor[c] // (hmax * 8)) for c in range(nc)], \
        [-(-H * info.v_samp_factor[c] // (vmax * 8)) for c in range(nc)]


def _device_classes(blocks, precision):
    """kind / reason / words of every block, as k_encode_seq decides them (relative offsets as absolute ones)"""
    for i in range(0, len(blocks), TILE):
        tb = blocks[i:i + TILE]
        nt = len(tb)
        for b in tb:
            n = len(b.bits)
            b.reason = "12-bit scan" if precision != 8 else "over 128 bits" if n > SLOT_BITS else \
                "ends a restart segment" if b.seg_end else ""
            b.kind = "fallback" if b.reason else "slot"
        end = tb[-1].off + len(tb[-1].bits)                         # s_off[nt]: the last block's end, no marker
        for j, b in enumerate(tb):
            o, n = b.off, len(b.bits)
            if b.kind == "fallback":
                e = o + n + (b.pad + 16 if b.seg_end else 0)
                b.words = [(w, "or") for w in range(o >> 5, -(-e // 32))]
                continue
            w = o >> 5 if (o & 31) and (j == 0 or tb[j - 1].kind == "fallback") else (o + 31) >> 5
            b.words = []
            while w * 32 < o + n:
                W = w * 32
                whole, m = o <= W, j
                while m < nt and tb[m].off < W + 32:
                    whole &= tb[m].kind == "slot"
                    m += 1
                if m == nt and end < W + 32:
                    whole = False
                b.words.append((w, "store" if whole else "or"))
                w += 1


def model_scans(jpeg, planes, info=None):
    """[ScanModel] of every scan of a sequential Huffman file whose final planes (per component (hib, wib, 64), natural
    order) are `planes`"""
    from mozjpeg_b200 import jpegtran as T
    if info is None:
        info = T.parse_source(jpeg)
    assert info.sof in (0xC0, 0xC1), "sequential Huffman files only"
    geom = _geometry(info)
    out = []
    for k in range(info.num_scans):
        sc = info.scans[k]
        mcus, per_row, slots, single = _scan_slots(info, sc, geom)
        comps = [sc.component_index[i] for i in range(sc.comps_in_scan)]
        dct = {c: code_table(info.huff[sc.dc_huff[i]]) for i, c in enumerate(comps)}
        act = {c: code_table(info.huff[sc.ac_huff[i]]) for i, c in enumerate(comps)}
        bim = len(slots)
        nblocks = mcus * bim
        seglen = sc.restart_interval * bim
        parts, markers, pos, pred = [], set(), 0, {c: 0 for c in comps}
        blocks = []
        for t in range(nblocks):
            m, s = divmod(t, bim)
            c, dx, dy = slots[s]
            if single:
                row, col = divmod(m, per_row)
            else:
                row, col = (m // per_row) * info.v_samp_factor[c] + dy, (m % per_row) * info.h_samp_factor[c] + dx
            if row >= planes[c].shape[0] or col >= planes[c].shape[1]:
                raise ValueError("dummy blocks are not modelled: use MCU-aligned sizes")
            if seglen and t % seglen == 0:
                pred = {cc: 0 for cc in comps}
            blk = planes[c][row, col]
            b = Block()
            b.t, b.comp, b.row, b.col, b.tile, b.j, b.off = t, c, row, col, t // TILE, t % TILE, pos
            b.bits = block_bits(blk, pred[c], dct[c], act[c])
            pred[c] = int(blk[0])
            parts.append(b.bits)
            pos += len(b.bits)
            b.seg_end = bool(seglen) and (t + 1) % seglen == 0 and t + 1 < nblocks
            b.pad = 0
            if b.seg_end:                                           # emit_restart (jchuff.c:668-686)
                b.pad = (8 - pos % 8) % 8
                parts.append("1" * b.pad + format(0xFFD0 + (t // seglen) % 8, "016b"))
                markers.add((pos + b.pad) // 8)
                pos += b.pad + 16
            blocks.append(b)
        parts.append("1" * ((8 - pos % 8) % 8))                     # flush_bits
        stream = "".join(parts)
        raw = int(stream, 2).to_bytes(len(stream) // 8, "big") if stream else b""
        data, src = bytearray(), []
        for i, x in enumerate(raw):
            data.append(x)
            src.append(i)
            if x == 0xFF and i not in markers and i - 1 not in markers:
                data.append(0)
                src.append(i)
        _device_classes(blocks, info.data_precision)
        out.append(ScanModel(k, info.data_precision, blocks, seglen, stream, markers, bytes(data), src))
    return out


def scan_bytes(jpeg, info=None):
    """the stuffed entropy-coded bytes of every scan of a file"""
    from decode_sync_cases import scan_data_end
    from mozjpeg_b200 import jpegtran as T
    if info is None:
        info = T.parse_source(jpeg)
    return [jpeg[info.scans[k].data_offset:scan_data_end(jpeg, info.scans[k].data_offset)] for k in range(info.num_scans)]


def first_difference(jpeg_want, jpeg_got, scans):
    """where two files of the same headers first differ, as locate() names it"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(jpeg_want)
    n = min(len(jpeg_want), len(jpeg_got))
    p = next((i for i in range(n) if jpeg_want[i] != jpeg_got[i]), n)
    for k in range(info.num_scans):
        lo = info.scans[k].data_offset
        if lo <= p < lo + len(scans[k].data) + 2:
            return "file byte %d: %s" % (p, scans[k].locate(p - lo))
    return "file byte %d, outside the entropy-coded data (%d vs %d bytes)" % (p, len(jpeg_want), len(jpeg_got))


# ---------------------------------------------------------------------------------------------------- the classes
LENGTHS = (6, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129)
STRUCTURE = ["span_5_words", "five_starts_in_word", "fb_between_slots_in_word", "fb_tile_first", "fb_tile_last",
             "slot_after_fb_mid_word", "tile_end_on_word_store", "tile_end_mid_word", "next_tile_phase_0",
             "next_tile_phase_nonzero", "tile_256_slot", "tile_256_fb", "last_tile_1", "last_tile_255"]
RESTART = ["rst_slot_sized_end", "rst_1block_segments", "marker_tile_first", "marker_tile_last"] + ["pad_%d" % i for i in range(8)]
STUFFING = ["ff_word_end", "ff_tile_edge", "ff_before_marker"]
ALL_CLASSES = ["len_%d" % n for n in LENGTHS] + ["slot128_phase_%d" % p for p in range(32)] + STRUCTURE + RESTART + STUFFING
# the classes a 12-bit scan (no slots: every block is a fallback block) can reach
TWELVE_CLASSES = ["tile_256_fb", "last_tile_1", "last_tile_255", "tile_end_mid_word", "next_tile_phase_nonzero",
                  "fb_tile_first", "fb_tile_last", "rst_1block_segments", "marker_tile_first", "marker_tile_last"] + \
                 ["pad_%d" % i for i in range(8)]


def scan_classes(s):
    """the boundary classes one ScanModel reaches"""
    out = set()
    bl = s.blocks
    eight = s.precision == 8
    for b in bl:
        n = len(b.bits)
        if eight and n in LENGTHS:
            out.add("len_%d" % n)
        if b.kind == "slot" and n == 128:
            out.add("slot128_phase_%d" % (b.off & 31))
        if b.off & 31 and (b.off + n - 1) // 32 - b.off // 32 + 1 >= 5:
            out.add("span_5_words")
        if b.seg_end:
            out.add("pad_%d" % b.pad)
            if eight and n <= SLOT_BITS:
                out.add("rst_slot_sized_end")
    if s.seglen == 1:
        out.add("rst_1block_segments")
    per_word = {}
    for b in bl:
        per_word.setdefault((b.tile, b.off >> 5), []).append(b)
    if any(len(v) >= 5 for v in per_word.values()):
        out.add("five_starts_in_word")
    for i in range(s.ntiles):
        tb = s.tile_blocks(i)
        last = tb[-1]
        end = last.off + len(last.bits) + (last.pad + 16 if last.seg_end else 0)
        if tb[0].kind == "fallback" and len(tb) > 1:
            out.add("fb_tile_first")
        if last.kind == "fallback" and len(tb) > 1:
            out.add("fb_tile_last")
        if len(tb) == TILE and all(b.kind == "slot" for b in tb):
            out.add("tile_256_slot")
        if len(tb) == TILE and all(b.kind == "fallback" for b in tb):
            out.add("tile_256_fb")
        if i + 1 < s.ntiles:
            if end % 32 == 0 and any(w == end // 32 - 1 and st == "store" for b in tb[-8:] for w, st in b.words):
                out.add("tile_end_on_word_store")
            if end % 32:
                out.add("tile_end_mid_word")
        if i:
            out.add("next_tile_phase_0" if tb[0].off % 32 == 0 else "next_tile_phase_nonzero")
        if i + 1 == s.ntiles and i:
            if len(tb) == 1:
                out.add("last_tile_1")
            if len(tb) == TILE - 1:
                out.add("last_tile_255")
        if last.seg_end:
            out.add("marker_tile_last")
        if tb[0].seg_end and len(tb) > 1 and (tb[0].off + len(tb[0].bits)) >> 5 == tb[0].off >> 5:
            out.add("marker_tile_first")
        for j, b in enumerate(tb):
            if j and b.kind == "slot" and b.off & 31 and tb[j - 1].kind == "fallback":
                out.add("slot_after_fb_mid_word")
            if 0 < j < len(tb) - 1 and b.kind == "fallback" and tb[j - 1].kind == "slot" and tb[j + 1].kind == "slot":
                a, c = tb[j - 1], tb[j + 1]
                if (a.off + len(a.bits) - 1) >> 5 == c.off >> 5:       # a's last bit and c's first bit in one word
                    out.add("fb_between_slots_in_word")
    raw = s.stream
    tile_first_bit = [s.blocks[i * TILE].off for i in range(1, s.ntiles)]
    for i in range(len(raw) // 8):
        if raw[8 * i:8 * i + 8] != "11111111" or i in s.markers or i - 1 in s.markers:
            continue
        if i % 4 == 3:
            out.add("ff_word_end")
        if any(8 * i < f < 8 * i + 8 for f in tile_first_bit):
            out.add("ff_tile_edge")
        b = s.block_at(8 * i)
        if b.seg_end and (b.off + len(b.bits) + b.pad) // 8 == i + 1:
            out.add("ff_before_marker")
    return out


def classes(scans):
    out = set()
    for s in scans:
        out |= scan_classes(s)
    return out


# ------------------------------------------------------------------------------------------- placed coefficients
# Under the standard tables a gray block with DC difference 0 and an immediate EOB is 6 bits; an AC (0,1) symbol adds 3
# and an (0,2) symbol 4; a DC difference of +-1 adds 2.  Chroma: 4 bits, 3, 5 and 1.  Every length from 6 up is
# reachable but 7 (luma) or 5 (chroma).
@functools.lru_cache(maxsize=None)
def std_lengths(chroma):
    """(DC code lengths by size, AC code lengths by symbol) of the standard tables, read back from a file"""
    from decode_sync_cases import encode
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(encode([np.zeros((2, 2, 64), np.int16)] + [np.zeros((1, 1, 64), np.int16)] * 2, "2x2", 16, 16))
    sc = info.scans[0]
    i = 1 if chroma else 0
    d, a = code_table(info.huff[sc.dc_huff[i]]), code_table(info.huff[sc.ac_huff[i]])
    return {s: v[1] for s, v in d.items()}, {s: v[1] for s, v in a.items()}


def recipe(L, chroma=False):
    """(DC difference size 0..2, (0,1) symbols, (0,2) symbols) of a block of exactly L bits, or None"""
    dl, al = std_lengths(chroma)
    a1, a2, eob = al[0x01] + 1, al[0x02] + 2, al[0x00]
    for k2 in range(64):
        for d in (0, 1, 2):
            r = L - dl[d] - d - k2 * a2
            if r < 0:
                continue
            if (r - eob) >= 0 and (r - eob) % a1 == 0 and (r - eob) // a1 + k2 <= 62:
                return d, (r - eob) // a1, k2
            if k2 <= 63 and r == (63 - k2) * a1:                 # position 63 filled: no EOB
                return d, 63 - k2, k2
    return None


def fill_block(blk, L, chroma, pred):
    """write a block of L bits into blk (natural order) after DC predictor pred; returns the block's DC"""
    rc = recipe(L, chroma)
    if rc is None:
        raise ValueError("no block of %d bits" % L)
    d, k1, k2 = rc
    blk[:] = 0
    dc = pred + (d * (-1 if pred > 0 else 1) if d else 0)
    blk[0] = dc
    k = 1
    for i in range(k2):
        blk[ZZ[k]] = (2, -3)[i % 2]
        k += 1
    for i in range(k1):
        blk[ZZ[k]] = (1, -1)[i % 2]
        k += 1
    return dc


def layout_blocks(layout, W, H):
    """per component (hib, wib) of an MCU-aligned image"""
    from decode_sync_cases import block_dims
    return block_dims(layout, W, H)


def scan_orders(layout, W, H, scans):
    """per scan, the (component, row, col) of every block in order t"""
    from decode_sync_cases import LAYOUTS
    f = LAYOUTS[layout]
    dims = layout_blocks(layout, W, H)
    hmax, vmax = max(h for h, _ in f), max(v for _, v in f)
    assert W % (8 * hmax) == 0 and H % (8 * vmax) == 0, "placed images are MCU-aligned"
    if scans == "multi" or len(f) == 1:
        return [[(c, r, x) for r in range(dims[c][0]) for x in range(dims[c][1])] for c in range(len(f))]
    order = []
    for my in range(H // (8 * vmax)):
        for mx in range(W // (8 * hmax)):
            for c, (h, v) in enumerate(f):
                order += [(c, my * v + y, mx * h + x) for y in range(v) for x in range(h)]
    return [order]


def place(layout, W, H, make_rule, scans="seq", restart=None):
    """planes whose blocks, in each scan's order t, have the lengths rule(t, n, bit offset mod 32) asks for (one
    make_rule() per scan) under the
    standard tables (restart: None or "<n>B", whose padding and markers move the offsets as k_scan_layout does)"""
    from decode_sync_cases import LAYOUTS
    dims = layout_blocks(layout, W, H)
    planes = [np.zeros((hb, wb, 64), np.int16) for hb, wb in dims]
    nmcu_blocks = sum(h * v for h, v in LAYOUTS[layout]) if scans != "multi" and len(dims) > 1 else 1
    ri = int(restart[:-1]) if restart else 0
    for order in scan_orders(layout, W, H, scans):
        rule = make_rule()
        seglen = ri * nmcu_blocks
        pos, pred = 0, {}
        n = len(order)
        for t, (c, r, x) in enumerate(order):
            if seglen and t % seglen == 0:
                pred = {}
            L = rule(t, n, pos % 32)
            pred[c] = fill_block(planes[c][r, x], L, c > 0, pred.get(c, 0))
            pos += L
            if seglen and (t + 1) % seglen == 0 and t + 1 < n:
                pos += (8 - pos % 8) % 8 + 16
    return planes


def to_phase(cur, p, lo=8):
    """a spacer length (6 or >= lo) that moves bit phase cur to p"""
    s = (p - cur) % 32
    return s if s == 6 or s >= lo else s + 32


def rule_lengths():
    """tile 0: every named length, a fallback then a mid-word slot block, the 128-bit slot block at all 32 phases, runs
    of 6-bit blocks, and an end on a word boundary; tile 1: fallback blocks first and last, ending mid-word; tile 2: 256
    slot blocks; tile 3: 256 fallback blocks of 129..160 bits (5 words at non-zero phases); then the last tile"""
    head = list(LENGTHS) + [8, 150, 6, 6, 6, 6, 6, 6, 9]
    state = {"plan": None}

    def rule(t, n, ph):
        tile, j = divmod(t, TILE)
        if tile == 0:
            if j < len(head):
                return head[j]
            plan = state["plan"]
            if plan is None:
                plan = state["plan"] = {"p": 0, "spaced": False}
            if plan["p"] < 32:
                if ph == plan["p"]:
                    plan["p"] += 1
                    return 128
                return to_phase(ph, plan["p"])
            if j == TILE - 1:
                return to_phase(ph, 0)
            return 6
        if tile == 1:
            if j in (0, TILE - 1):
                return 200 + j % 7
            if j == 1:
                return to_phase(ph, 5)
            return (6, 40, 8, 129, 66, 100)[j % 6]
        if tile == 2:
            return 6
        if tile == 3:
            return 129 + j % 32
        return (6, 8, 128, 131)[j % 4]
    return rule


def rule_restart():
    """restart segments of 4 blocks [x, y, a, b]: a ends 1 bit into a word, b (6 bits) ends the segment, so a slot block,
    the fallback block b with its marker and the next segment's first slot block share one word; the segment-ending
    blocks' lengths cycle through all eight paddings"""
    def rule(t, n, ph):
        k = t % 4
        if k == 0:
            return 6
        if k == 1:
            return 8 + (t // 4) % 8
        if k == 2:
            return to_phase(ph, 1, lo=33)
        return (6, 8, 9)[(t // 4) % 3]
    return rule


def rule_every_block_restart():
    """-restart 1B: every block but the last ends a segment; lengths 8..15 give every padding, with a few long blocks"""
    def rule(t, n, ph):
        return 250 if t % 97 == 5 else 8 + t % 8 + 8 * ((t // 8) % 3)
    return rule


def rule_tiles_on_words():
    """4:2:0 MCUs: every tile ends on a word boundary or, every other tile, 12 bits into one; 128-bit blocks and
    fallback blocks of both tables at several phases"""
    def rule(t, n, ph):
        j = t % TILE
        if j == TILE - 1:
            return to_phase(ph, 0 if (t // TILE) % 2 == 0 else 12)
        return (128, 6, 11, 129, 33, 64, 97, 8, 140, 128, 31, 95)[t % 12] if t % 12 else 128
    return rule


# (id, layout, width, height, rule, scans, restart): MCU-aligned sizes; the tile counts are set by the sizes
PLACED = {
    "gray_lengths": ("gray", 41 * 8, 25 * 8, rule_lengths, "seq", None),          # 1025 blocks: last tile of 1
    "gray_lengths_255": ("gray", 59 * 8, 13 * 8, rule_lengths, "seq", None),      # 767 blocks: last tile of 255
    "gray_restart4": ("gray", 40 * 8, 20 * 8, rule_restart, "seq", "4B"),
    "gray_restart1": ("gray", 32 * 8, 17 * 8, rule_every_block_restart, "seq", "1B"),
    "420_tiles": ("2x2", 32 * 16, 12 * 16, rule_tiles_on_words, "seq", None),
    "420_restart": ("2x2", 16 * 16, 6 * 16, rule_restart, "seq", "2B"),
    "420_multi": ("2x2", 32 * 16, 12 * 16, rule_lengths, "multi", None),
}


@functools.lru_cache(maxsize=None)
def placed_planes(pid):
    layout, W, H, rule, scans, restart = PLACED[pid]
    return tuple(place(layout, W, H, rule, scans, restart))


def ff_planes():
    """the adversarial suite's mostly-0xFF gray plane, five tiles of it, with a DC difference of 1023 on every tile's
    first block (whose DC code 11111110 and value bits carry the previous block's trailing one-bits across the tile
    edge) and of 1 in every tile (so that tile edges fall inside bytes)"""
    import adversarial_cases as AC
    pl = AC.ff_plane(64, 20)[0].reshape(-1, 64).copy()
    pl[::TILE, 0] = 1023
    pl[100::TILE, 0] = 1
    return (pl.reshape(20, 64, 64),)


def coef_params(layout, W, H, variant, scans, restart):
    """the parameter block of a coefficient encode: variant "fixed" (-revert, standard tables), "opt" (-optimize:
    per-image tables) or "12" (12-bit, optimal tables)"""
    from decode_sync_cases import params
    return params(layout, W, H, precision=12 if variant == "12" else 8, optimize=variant == "opt", restart=restart, scans=scans)


# coefficient cases: (id, planes source, variant); a source is a PLACED id or "ff" / "ff_restart1"
COEF_CASES = [(p + ":" + v, p, v) for p in PLACED for v in ("fixed", "opt", "12")] + \
             [("ff:fixed", "ff", "fixed"), ("ff_restart1:fixed", "ff_restart1", "fixed")]


def coef_source(src):
    """(layout, W, H, scans, restart, planes) of a coefficient planes source"""
    if src.startswith("ff"):
        pl = ff_planes()
        return "gray", pl[0].shape[1] * 8, pl[0].shape[0] * 8, "seq", "1B" if src == "ff_restart1" else None, pl
    layout, W, H, _, scans, restart = PLACED[src]
    return layout, W, H, scans, restart, placed_planes(src)


@functools.lru_cache(maxsize=None)
def coef_case(cid):
    """(oracle file, planes, params) of a COEF_CASES id"""
    from oracle import oracle as O
    _, src, variant = next(c for c in COEF_CASES if c[0] == cid)
    layout, W, H, scans, restart, pl = coef_source(src)
    p = coef_params(layout, W, H, variant, scans, restart)
    return O.oracle_encode_coefs(p, list(pl)), pl, p


def ref_switches(cid):
    """jpegtran switches that re-encode a plain carrier of the case's planes to the case's file"""
    _, src, variant = next(c for c in COEF_CASES if c[0] == cid)
    _, _, _, scans, restart, _ = coef_source(src)
    return ["-revert"] + (["-optimize"] if variant == "opt" else []) + (["-restart", restart] if restart else []), scans


# --------------------------------------------------------------------------------------------------- pixel input
def noise_ramps(seed, w, h):
    """8x8 blocks in columns: noise whose amplitude ramps across the image, beside flat blocks"""
    rng = np.random.default_rng(seed)
    x = np.arange(w)[None, :]
    amp = ((np.arange(h)[:, None] // 8) * 3 + (x // 8) * 5) % 40 + 2
    noise = rng.normal(0, 1, (h, w)) * amp
    base = 128 + 40 * np.sin(x / 23.0)
    flat = ((x // 8) % 3 == 1) | ((np.arange(h)[:, None] // 8) % 5 == 2)
    im = np.where(flat, np.round(base / 8) * 8, base + noise)
    im = np.clip(np.round(im), 0, 255).astype(np.uint8)
    return np.stack([im, np.roll(im, 8, 1), np.roll(im, 16, 0)], axis=2)


# (id, seed, width, height, gray, quality, walk, restart): walk "symrec" (default trellis), "loops", "scans_in_trellis",
# "q_opt", "eob_opt" (generic trellis rounds: final coefficient planes) or "notrellis" (plain-quantized planes)
PIXEL_CASES = [
    ("gray_q95_symrec", 3, 256, 136, True, 95, "symrec", None),
    ("gray_q100_symrec_rst", 4, 256, 96, True, 100, "symrec", "4B"),
    ("420_q90_symrec", 5, 256, 96, False, 90, "symrec", None),
    ("gray_q95_loops", 6, 256, 136, True, 95, "loops", None),
    ("gray_q100_scans_in_trellis", 7, 256, 96, True, 100, "scans_in_trellis", "5B"),
    ("420_q85_q_opt", 8, 256, 96, False, 85, "q_opt", None),
    ("gray_q98_eob_opt", 9, 256, 136, True, 98, "eob_opt", "1B"),
    ("gray_q97_notrellis", 10, 256, 136, True, 97, "notrellis", None),
]
PIXEL = {c[0]: c for c in PIXEL_CASES}


def pixel_params(pid):
    import mozjpeg_b200 as mj
    _, seed, w, h, gray, q, walk, restart = PIXEL[pid]
    sw = ["-baseline", "-quality", str(q)] + (["-grayscale"] if gray else ["-sample", "2x2"]) + \
        (["-restart", restart] if restart else []) + (["-notrellis"] if walk == "notrellis" else [])
    p = mj.params_from_switches(sw, w, h, 3)
    if walk == "loops":
        p.trellis_num_loops = 2
    elif walk == "scans_in_trellis":
        p.use_scans_in_trellis = 1
    elif walk == "q_opt":
        p.trellis_q_opt = 1
    elif walk == "eob_opt":
        p.trellis_eob_opt = 1
    return p


def pixel_image(pid):
    _, seed, w, h, _, _, _, _ = PIXEL[pid]
    return noise_ramps(seed, w, h)


def pixel_walk(pid):
    walk = PIXEL[pid][6]
    return {"symrec": "symrec", "notrellis": "dense"}.get(walk, "generic_rounds")


@functools.lru_cache(maxsize=None)
def pixel_case(pid):
    """(oracle file, final planes, params) of a PIXEL_CASES id"""
    from oracle import oracle as O
    p = pixel_params(pid)
    r = O.oracle_encode(p, pixel_image(pid), want_debug=True)
    d = r.dbg
    planes = tuple(np.ascontiguousarray(d["final"][c][:d["hib"][c], :d["wib"][c]]) for c in range(p.num_components))
    return r.jpeg, planes, p


# the classes each walk must reach (the pixel walks: what the families above reach, found by search)
_PIXEL_REACHED = {"len_127", "len_128", "len_129", "span_5_words", "fb_tile_first", "fb_tile_last", "slot_after_fb_mid_word",
                  "tile_end_mid_word", "next_tile_phase_nonzero", "rst_slot_sized_end", "marker_tile_last", "ff_word_end",
                  "ff_before_marker"} | {"pad_%d" % i for i in range(8)}
WALK_CLASSES = {
    "dense": set(ALL_CLASSES),
    "dense12": set(TWELVE_CLASSES),
    "symrec": _PIXEL_REACHED,
    "generic_rounds": _PIXEL_REACHED | {"rst_1block_segments", "tile_256_fb"},
}


def case_walk(cid):
    """the walk a case of either list runs on the device"""
    if cid in PIXEL:
        return pixel_walk(cid)
    return "dense12" if cid.endswith(":12") else "dense"


def case(cid):
    """(oracle file, planes, params) of a case of either list"""
    return pixel_case(cid) if cid in PIXEL else coef_case(cid)


ALL_CASES = [c[0] for c in COEF_CASES] + [c[0] for c in PIXEL_CASES]
