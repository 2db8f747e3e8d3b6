"""Sources of the progressive-decode model tests (tests/test_progressive_model.py): a serial model of the decode of
progressive Huffman files (SOF2) with the device's rules, a scan writer that turns token lists back into entropy-coded
bytes, scans constructed with it at the edges of the four scan kinds, and per-scan damage of small progressive files.

The model restates decode_mcu_DC_first, decode_mcu_AC_first, decode_mcu_DC_refine and decode_mcu_AC_refine
(jdphuff.c) over build_decode_batch's restart segments, with the device's semantics (DESIGN §8): an invalid code or
bits needed past a segment's end is status 1 in every scan kind, and so is a DC refinement segment with fewer bits than
blocks; a first-scan value past a band that ends before 63 is status 2, not written, and the decode goes on; a
refinement value past such a band is status 2 and a refinement symbol of size other than 1 is status 4, and either
ends its segment with the earlier blocks kept; a run past 63 writes position 63; whatever follows a segment's last
block is ignored.  Every generator is seeded, so a failing case reproduces."""
import re
import struct

import numpy as np

import adversarial_cases as AC
import decode_sync_cases as S
import progressive_cases as P

ZZ = np.asarray(AC.ZZ)
# the device's messages per status bit, in the order encoder.cu checks them
STATUS_WORDS = {1: "an invalid Huffman code, or too few bits for a segment's MCUs",
                2: "a coefficient past the end of its scan's spectral band",
                4: "an AC refinement symbol whose size is not 1"}
# refusals where the reference decodes on without a warning (b200jpeg.h, DESIGN §8): a documented difference
DOCUMENTED = ("a second first scan", STATUS_WORDS[2])
KINDS = ("dc_first", "dc_refine", "ac_first", "ac_refine")


def kind(sc):
    return ("dc_" if sc.Ss == 0 else "ac_") + ("refine" if sc.Ah else "first")


class Refusal(Exception):
    """the device refuses the file: status bits of the decode kernels (1, 2, 4), or 0 and the host's words"""

    def __init__(self, status, words, planes=None):
        super().__init__(words)
        self.status, self.words, self.planes = status, words, planes

# --------------------------------------------------------------------------------------------------------- bit reader
class _Dead(Exception):
    pass


class _Reader:
    """one restart segment's unstuffed bytes, read MSB first with zero bits behind them (the device's zero words);
    log: a list that receives the tokens read, ("h", tkey, symbol, extra value, extra length) or ("b", value, n)"""

    def __init__(self, data, log=None):
        self.nbits = 8 * len(data)
        self.total = self.nbits + 32
        self.bits = int.from_bytes(data, "big") << 32
        self.pos = 0
        self.log = log

    def _peek(self, n):
        return (self.bits >> (self.total - self.pos - n)) & ((1 << n) - 1) if n else 0

    def symbol(self, codes, tkey, extra_of):
        """a Huffman symbol and its extra bits (extra_of(symbol) of them); _Dead for a code no entry matches or one that
        ends past the segment"""
        code = 0
        for ln in range(1, 17):
            code = (code << 1) | ((self.bits >> (self.total - 1 - self.pos - ln + 1)) & 1)
            sym = codes.get((ln, code))
            if sym is not None:
                break
        else:
            raise _Dead
        n = extra_of(sym)
        if self.pos + ln + n > self.nbits:
            raise _Dead
        self.pos += ln
        x = self._peek(n)
        self.pos += n
        if self.log is not None:
            self.log.append(("h", tkey, sym, x, n))
        return sym, x

    def raw(self, n):
        if self.pos + n > self.nbits:
            raise _Dead
        x = self._peek(n)
        self.pos += n
        if self.log is not None and n:
            self.log.append(("b", x, n))
        return x


# ---------------------------------------------------------------------------------------------------------- the model
def _s16(v):
    return ((int(v) + 32768) & 0xFFFF) - 32768


def _host_checks(jpeg):
    """parse_source and check_progression (source.cpp): the parsed headers, or Refusal with the host's words"""
    from mozjpeg_b200 import jpegtran as T
    try:
        info = T.parse_source(jpeg)
    except ValueError as e:
        raise Refusal(0, str(e))
    if info.sof != 0xC2:
        raise ValueError("progressive files only")
    cb = [[-1] * 64 for _ in range(4)]
    for n in range(info.num_scans):
        sc = info.scans[n]
        dc = sc.Ss == 0
        bad = sc.Se != 0 if dc else (sc.Ss > sc.Se or sc.Se >= 64 or sc.comps_in_scan != 1)
        if (sc.Ah != 0 and sc.Al != sc.Ah - 1) or sc.Al > 13:
            bad = True
        if bad:
            raise Refusal(0, f"scan {n}: bad progression parameters")
        for i in range(sc.comps_in_scan):
            c = cb[sc.component_index[i]]
            if not dc and c[0] < 0:
                raise Refusal(0, f"scan {n}: bogus progression: AC scan of component {sc.component_index[i]} before its DC scan")
            for k in range(sc.Ss, sc.Se + 1):
                if sc.Ah != max(c[k], 0):
                    raise Refusal(0, f"scan {n}: bogus progression: Ah={sc.Ah} for coefficient {k}")
                if sc.Ah == 0 and c[k] >= 0:
                    raise Refusal(0, f"scan {n}: bogus progression: a second first scan of coefficient {k}")
                c[k] = sc.Al
    return info


def _segments(jpeg, info, k):
    sc = info.scans[k]
    mcus, _, _ = S.scan_layout(info, sc)
    ri = sc.restart_interval
    nseg = -(-mcus // ri) if ri else 1
    try:
        segs = S.unstuff(jpeg, sc.data_offset, sc.data_offset + sc.data_size, ri, nseg)
    except S.Refused as e:                              # the host's words: "scan <k> ends after ..." / "restart marker ..."
        raise Refusal(0, str(e).replace("scan ends after", "ends after"))
    return segs, mcus, ri


def decode(jpeg: bytes, upto=None, log=None):
    """The planes the device decode makes of a progressive file, or Refusal (status bits with the planes as the device
    leaves them, or the host's words).  Scans are taken in file order, which after the progression check gives the
    device's order: a coefficient's refinements follow its first scan, and scans of one level touch disjoint
    coefficients.  upto: decode scans [0, upto) only.  log: a dict that receives per scan the token lists of its
    segments."""
    info = _host_checks(jpeg)
    hmax, vmax, wib, hib = S._geometry(info)
    nc = info.num_components
    out = [np.zeros((hib[c], wib[c], 64), np.int16) for c in range(nc)]
    status = 0
    scans = range(info.num_scans if upto is None else upto)
    parts = [(k, *_segments(jpeg, info, k)) for k in scans]          # the host unstuffs every scan before any decode
    for k, segs, mcus, ri in parts:
        sc = info.scans[k]
        _, per_row, slots = S.scan_layout(info, sc)
        comps = [sc.component_index[i] for i in range(sc.comps_in_scan)]
        knd = kind(sc)
        dct = {c: S._codes(info.huff[sc.dc_huff[i]]) for i, c in enumerate(comps)} if knd == "dc_first" else {}
        act = {c: S._codes(info.huff[sc.ac_huff[i]]) for i, c in enumerate(comps)} if knd[:3] == "ac_" else {}
        tk = {c: ((0, sc.dc_tbl_no[i]), (1, sc.ac_tbl_no[i])) for i, c in enumerate(comps)}
        mx = {c: (1 if len(comps) == 1 else info.h_samp_factor[c]) for c in comps}
        my = {c: (1 if len(comps) == 1 else info.v_samp_factor[c]) for c in comps}
        logs = []
        for sg, data in enumerate(segs):
            toks = [] if log is not None else None
            logs.append(toks)
            rd = _Reader(data, toks)
            nmcu = min(ri, mcus - sg * ri) if ri else mcus
            m0 = sg * ri if ri else 0
            blocks = []
            for m in range(m0, m0 + nmcu):
                for c, dx, dy in slots:
                    col, row = (m % per_row) * mx[c] + dx, (m // per_row) * my[c] + dy
                    blocks.append((c, out[c][row, col] if col < wib[c] and row < hib[c] else None))
            try:
                if knd == "dc_first":
                    _dc_first(rd, blocks, dct, tk, sc.Al)
                elif knd == "dc_refine":
                    if rd.nbits < len(blocks):
                        status |= 1                     # k_dec_dc_refine: the blocks with a bit still take it
                    for b, (c, blk) in enumerate(blocks[:rd.nbits]):
                        if rd.raw(1) and blk is not None:
                            blk[0] = _s16((int(blk[0]) & 0xFFFF) | (1 << sc.Al))
                elif knd == "ac_first":
                    status |= _ac_first(rd, blocks, act, tk, sc)
                else:
                    status |= _ac_refine(rd, blocks, act, tk, sc)
            except _Dead:
                status |= 1
        if log is not None:
            log[k] = logs
    if status:
        raise Refusal(status, STATUS_WORDS[status & -status], out)
    return out


def _dc_first(rd, blocks, dct, tk, Al):
    pred = {}
    for c, blk in blocks:
        s, x = rd.symbol(dct[c], tk[c][0], lambda sym: sym)
        pred[c] = pred.get(c, 0) + S._extend(x, s)
        if blk is not None:
            blk[0] = _s16(pred[c] << Al)


def _ac_first(rd, blocks, act, tk, sc):
    status, b = 0, 0
    while b < len(blocks):
        c, blk = blocks[b]
        k, done = sc.Ss, 1
        while k <= sc.Se:
            sym, x = rd.symbol(act[c], tk[c][1], lambda sym: sym & 15 if (sym & 15 or sym >> 4 == 15) else sym >> 4)
            r, s = sym >> 4, sym & 15
            if s:
                k += r
                z = min(k, 63)
                if z > sc.Se:
                    status |= 2                         # past a band that ends before 63: not written
                else:
                    blk[ZZ[z]] = _s16(S._extend(x, s) << sc.Al)
                k += 1
            elif r == 15:
                k += 16
            else:
                done = (1 << r) + x
                break
        b += done                                       # an EOB run past the segment's last block ends the segment
    return status


def _ac_refine(rd, blocks, act, tk, sc):
    Ss, Se, Al = sc.Ss, sc.Se, sc.Al
    p1, m1 = 1 << Al, -(1 << Al)
    eobrun = 0
    for c, blk in blocks:
        nz = [blk[ZZ[p]] != 0 if Ss <= p <= Se else False for p in range(64)]
        inc, newnz, k, err = set(), {}, Ss, 0
        try:
            if eobrun == 0:
                while k <= Se:
                    sym, x = rd.symbol(act[c], tk[c][1], lambda sym: 0 if sym & 15 or sym >> 4 == 15 else sym >> 4)
                    r, s = sym >> 4, sym & 15
                    neg = False
                    if s:
                        if s != 1:
                            err = 4
                            break
                        neg = not rd.raw(1)
                    elif r != 15:
                        eobrun = (1 << r) + x
                        break
                    zeros = [p for p in range(k, Se + 1) if not nz[p]]
                    target = zeros[r] if len(zeros) > r else Se + 1
                    before = [p for p in range(k, min(target, Se + 1)) if nz[p]]
                    bits = rd.raw(len(before))
                    inc |= {p for i, p in enumerate(before) if (bits >> (len(before) - 1 - i)) & 1}
                    k = target
                    if s:
                        if k > Se and Se < 63:
                            err = 2
                            break
                        newnz[min(k, 63)] = neg
                    k += 1
            if not err and eobrun > 0:
                rest = [p for p in range(k, Se + 1) if nz[p]]
                bits = rd.raw(len(rest))
                inc |= {p for i, p in enumerate(rest) if (bits >> (len(rest) - 1 - i)) & 1}
                eobrun -= 1
        except _Dead:
            err = 1
        if err:
            return err                                  # the segment ends; its earlier blocks keep their values
        for p in range(64):
            n = ZZ[p]
            if p in newnz:
                blk[n] = m1 if newnz[p] else p1
            elif p in inc and not (int(blk[n]) & p1):
                v = int(blk[n])
                blk[n] = _s16(v + (p1 if v >= 0 else m1))
    return 0


def verdict(jpeg: bytes):
    """("ok", planes), ("status", bits, planes) or ("host", words)"""
    try:
        return ("ok", decode(jpeg))
    except Refusal as e:
        return ("status", e.status, e.planes) if e.status else ("host", e.words)


# ------------------------------------------------------------------------------------------------------ scan writer
def _dht(tables):
    """one DHT segment of {(class, id): (bits[0..16], huffval)}"""
    body = b""
    for (cls, tid), (bits, vals) in sorted(tables.items()):
        body += bytes([cls << 4 | tid]) + bytes(bits[1:17]) + bytes(vals)
    return b"\xff\xc4" + struct.pack(">H", 2 + len(body)) + body


def tables_for(segments):
    """per table key, the optimal table (jpeg_gen_optimal_table) of the symbols the token lists use"""
    freq = {}
    for toks in segments:
        for t in toks:
            if t[0] == "h":
                freq.setdefault(t[1], np.zeros(256, np.int64))[t[2]] += 1
    return {key: AC.gen_optimal_table(f)[:2] for key, f in freq.items()}


def _codes_of(bits, vals):
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln]):
            out[vals[k]] = (code, ln)
            code += 1
            k += 1
        code <<= 1
    return out


def write_scan(segments, tables) -> bytes:
    """entropy-coded bytes of a scan from per-segment token lists: each segment padded with 1-bits to a byte, 0xFF
    stuffed, RSTn between segments.  tables: {(class, id): (bits, huffval)}"""
    codes = {key: _codes_of(*t) for key, t in tables.items()}
    out = b""
    for sg, toks in enumerate(segments):
        acc, n = 0, 0
        for t in toks:
            if t[0] == "h":
                code, ln = codes[t[1]][t[2]]
                acc, n = (acc << ln) | code, n + ln
                acc, n = (acc << t[4]) | t[3], n + t[4]
            else:
                acc, n = (acc << t[2]) | t[1], n + t[2]
        pad = -n % 8
        acc, n = (acc << pad) | ((1 << pad) - 1), n + pad
        data = acc.to_bytes(n // 8, "big") if n else b""
        out += data.replace(b"\xff", b"\xff\x00")
        if sg + 1 < len(segments):
            out += bytes([0xFF, 0xD0 + (sg & 7)])
    return out


def splice(carrier: bytes, scans) -> bytes:
    """carrier with the entropy-coded data of some scans replaced: {scan index: (data bytes, DHT bytes or b"")}, the
    DHT written in front of the scan's SOS"""
    segs = P.segments(carrier)
    out, n = [carrier[:2]], 0
    for m, a, b in segs:
        if m == 0xDA and n in scans:
            data, dht = scans[n]
            hl = struct.unpack(">H", carrier[a + 2:a + 4])[0]
            out += [dht, carrier[a:a + 2 + hl], data]
        else:
            out.append(carrier[a:b])
        n += m == 0xDA
    return b"".join(out) + b"\xff\xd9"


def file_tables(info, k):
    """{(class, id): (bits, huffval)} of the tables scan k uses"""
    sc = info.scans[k]
    out = {}
    for i in range(sc.comps_in_scan if not (sc.Ss == 0 and sc.Ah) else 0):
        for cls, pool, tid in ((0, sc.dc_huff[i], sc.dc_tbl_no[i]),) if sc.Ss == 0 else ((1, sc.ac_huff[i], sc.ac_tbl_no[i]),):
            h = info.huff[pool]
            n = sum(h.bits[1:17])
            out[(cls, tid)] = (list(h.bits[:17]), list(h.huffval[:n]))
    return out


def rewrite(jpeg: bytes) -> bytes:
    """the file with every scan's data written again from the tokens the model reads (the writer's round trip)"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(jpeg)
    log = {}
    decode(jpeg, log=log)
    return splice(jpeg, {k: (write_scan(log[k], file_tables(info, k)), b"") for k in log})


def replace_scan(carrier: bytes, k: int, segments) -> bytes:
    """carrier with scan k's data written from the token lists, behind a DHT of their own tables"""
    tabs = tables_for(segments)
    return splice(carrier, {k: (write_scan(segments, tabs), _dht(tabs) if tabs else b"")})


# --------------------------------------------------------------------------------------------------- token helpers
def tok(sym, x=0, n=0, key=(1, 0)):
    """a Huffman symbol of table key with n extra bits x"""
    return ("h", key, sym, x, n)


def B(x, n=1):
    return ("b", x, n)


def ONES(n=16):
    """n one-bits: never a code of a table jpeg_gen_optimal_table makes (it keeps the all-ones code free)"""
    return ("b", (1 << n) - 1, n)


def _value_bits(v):
    s = int(abs(v)).bit_length()
    return s, (v if v >= 0 else v + (1 << s) - 1)


def dc_sym(diff, key=(0, 0)):
    s, x = _value_bits(diff)
    return tok(s, x, s, key)


def ac_sym(r, v):
    s, x = _value_bits(v)
    return tok(r << 4 | s, x, s)


def eob(r, x=0):
    return tok(r << 4, x, r)


def refine_tokens(before, Ss, Se, program, seed=0):
    """Tokens of one AC refinement segment over the blocks of `before` ([n][64] natural order, the coefficients the
    scan starts from).  program: per block a list of ops, ("v", r, negative[, size]) a new value after r zeros (size:
    the symbol's size, 1 unless a refusal is wanted), ("zrl",), ("eob", r, x) an EOB run of 2^r + x blocks starting
    here; blocks inside a run take no ops.  Correction bits are seeded.  Walks the band as decode_mcu_AC_refine does."""
    rng = np.random.default_rng(seed)
    toks, run = [], 0
    for b, ops in enumerate(program):
        nz = [Ss <= p <= Se and before[b][ZZ[p]] != 0 for p in range(64)]

        def corr(ps):
            for _ in ps:
                toks.append(B(int(rng.integers(0, 2))))
        k = Ss
        if run:
            assert not ops, b
            corr([p for p in range(k, Se + 1) if nz[p]])
            run -= 1
            continue
        for op in ops:
            if op[0] == "eob":
                toks.append(eob(op[1], op[2]))
                corr([p for p in range(k, Se + 1) if nz[p]])
                run = (1 << op[1]) + op[2] - 1
                break
            r = 15 if op[0] == "zrl" else op[1]
            if op[0] == "zrl":
                toks.append(tok(0xF0))
            else:
                toks.append(tok(r << 4 | (op[3] if len(op) > 3 else 1), 0 if op[2] else 1, 1))
            passed = []
            while k <= Se:
                if nz[k]:
                    passed.append(k)
                else:
                    if r == 0:
                        break
                    r -= 1
                k += 1
            corr(passed)
            k += 1
    return toks


# -------------------------------------------------------------------------------------------------------- carriers
def script_params(layout, W, H, script, precision=8, restart=None):
    """b200jpeg_params of a progressive file with the given script [(components, Ss, Se, Ah, Al)]"""
    p = S.params(layout, W, H, precision=precision, restart=restart, scans="prog")
    p.num_scans = len(script)
    for k, (comps, ss, se, ah, al) in enumerate(script):
        s = p.scan_info[k]
        s.comps_in_scan, s.Ss, s.Se, s.Ah, s.Al = len(comps), ss, se, ah, al
        for i, c in enumerate(comps):
            s.component_index[i] = c
    return p


def carrier(planes, layout, W, H, script, precision=8, restart=None) -> bytes:
    from oracle import oracle as O
    return O.oracle_encode_coefs(script_params(layout, W, H, script, precision, restart), planes)


SCRIPT_FULL = [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 1), ((0,), 1, 63, 1, 0)]
SCRIPT_SPLIT = [((0,), 0, 0, 0, 0), ((0,), 1, 9, 0, 1), ((0,), 10, 63, 0, 1), ((0,), 1, 9, 1, 0), ((0,), 10, 63, 1, 0)]


def _refine_plane(wb, hb, seed, dense=False, last_count=None):
    """a gray plane whose AC values are mostly +-2..5 (nonzero after an Al 1 first scan) at seeded zigzag positions;
    dense: every AC position nonzero; last_count: the last block holds values at zigzag 1 .. last_count"""
    rng = np.random.default_rng(seed)
    pl = np.zeros((hb * wb, 64), np.int16)
    pl[:, 0] = rng.integers(-30, 31, hb * wb)
    for b in range(hb * wb):
        ks = np.arange(1, 64) if dense else rng.choice(np.arange(1, 64), int(rng.integers(3, 12)), replace=False)
        pl[b, ZZ[ks]] = rng.choice([-5, -3, -2, 2, 3, 4], len(ks))
    if last_count is not None:
        pl[-1, 1:] = 0
        pl[-1, ZZ[np.arange(1, last_count + 1)]] = 3
    return [pl.reshape(hb, wb, 64)]


def _state(jpeg, k):
    """per block (raster order) the coefficients component 0 holds before scan k"""
    return decode(jpeg, upto=k)[0].reshape(-1, 64)


def _with_refine(pl, script, k, program_of, W, H, restart=None, seed=0):
    """(file, carrier) with the AC refinement scan k of a gray carrier written from program_of(before, Ss, Se), per
    block its ops (refine_tokens), cut into restart segments of `restart` ("<n>B") blocks"""
    car = carrier(pl, "gray", W, H, script, restart=restart)
    from mozjpeg_b200 import jpegtran as T
    sc = T.parse_source(car).scans[k]
    before = _state(car, k)
    prog = program_of(before, sc.Ss, sc.Se)
    assert len(prog) == len(before), (len(prog), len(before))
    n = int(restart[:-1]) if restart else len(prog)
    segs = [refine_tokens(before[b:b + n], sc.Ss, sc.Se, prog[b:b + n], seed + b) for b in range(0, len(prog), n)]
    return replace_scan(car, k, segs), car


def _zeros(before_blk, k, Ss, Se):
    return [p for p in range(max(k, Ss), Se + 1) if before_blk[ZZ[p]] == 0]


def _run_to_end(n):
    """ops for the first of n blocks that puts all n in one EOB run (EOBr with r = floor(log2 n))"""
    r = n.bit_length() - 1
    return [("eob", r, n - (1 << r))]


# (id, expected verdict): "ok", a status bit (1, 2, 4) or "host: <words>"
CONSTRUCTED = {
    "refine_zrl_over_nonzero": "ok",
    "refine_zrl_past_se": "ok",
    "refine_value_at_se_split": "ok",
    "refine_value_at_63": "ok",
    "refine_value_past_63_overwrites": "ok",
    "refine_value_past_63_dense": "ok",
    "refine_mid_block_eobr": "ok",
    "refine_every_eobr": "ok",
    "refine_eobrun_overshoots_segment": "ok",
    "refine_split_bands_ss10": "ok",
    "refine_dense_blocks": "ok",
    "refine_size_2": 4,
    "refine_size_15": 4,
    "refine_value_past_se": 2,
    "refine_cut_in_eob_tail": 1,
    "refine_ends_on_last_correction_bit": "ok",
    "refine_empty_segment": 1,
    "refine_invalid_code": 1,
    "ac_first_value_past_se": 2,
    "ac_first_value_at_se": "ok",
    "ac_first_run_past_63": "ok",
    "ac_first_eobrun_past_end_garbage": "ok",
    "ac_first_eobrun_past_end_garbage_restart": "ok",
    "ac_first_empty_segment": 1,
    "ac_first_invalid_code": 1,
    "dc_refine_8n_blocks_in_n_bytes": "ok",
    "dc_refine_8n_plus_1_blocks": 1,
    "dc_refine_empty_segment": 1,
    "dc_first_al13_12bit_negative": "ok",
    "dc_first_empty_segment": 1,
    "dc_first_invalid_code": 1,
    "second_first_scan": "host: a second first scan",
}


def constructed(cid):
    """(file, carrier it was built on) of a constructed case"""
    W, H = 64, 16                                                           # 8 x 2 blocks
    if cid == "refine_zrl_over_nonzero":
        pl = _refine_plane(8, 2, 1)
        for b in range(16):                                                 # nonzeros among the first 16 zeros
            pl[0].reshape(-1, 64)[b, ZZ[[2, 5, 9, 14, 20]]] = 2
        return _with_refine(pl, SCRIPT_FULL, 2, lambda bf, ss, se: [[("zrl",), ("v", 0, False), ("zrl",)] + _run_to_end(16)]
                            + [[] for _ in range(15)], W, H)
    if cid == "refine_zrl_past_se":                                         # band 1-9: fewer than 16 zeros left
        pl = _refine_plane(8, 2, 2)
        pl[0].reshape(-1, 64)[:, ZZ[1:10]] = [0, 2, 0, 0, -3, 0, 0, 0, 0]
        return _with_refine(pl, SCRIPT_SPLIT, 3, lambda bf, ss, se: [[("v", 0, True), ("zrl",)] for _ in range(16)], W, H)
    if cid in ("refine_value_at_se_split", "refine_value_past_se", "refine_value_at_63", "refine_value_past_63_overwrites"):
        split = cid.endswith("split") or cid == "refine_value_past_se"
        pl = _refine_plane(8, 2, 3)
        blk = pl[0].reshape(-1, 64)
        blk[:, ZZ[[1, 3, 4, 6, 7, 8, 9]]] = 0                               # zeros in the 1-9 band, zigzag 9 among them
        blk[:, ZZ[63]] = 3 if cid == "refine_value_past_63_overwrites" else 0
        extra = 1 if cid in ("refine_value_past_se", "refine_value_past_63_overwrites") else 0

        def prog(bf, ss, se):                                               # one value onto the last zero, or past it
            out = []
            for b in range(16):
                z = len(_zeros(bf[b], ss, ss, se)) - 1 + extra
                out.append([("zrl",)] * (z // 16) + [("v", z % 16, b % 2 == 1)])
            return out
        return _with_refine(pl, SCRIPT_SPLIT if split else SCRIPT_FULL, 3 if split else 2, prog, W, H)
    if cid == "refine_value_past_63_dense":                                # no zero at all: the value goes to 63
        pl = _refine_plane(8, 2, 4, dense=True)
        return _with_refine(pl, SCRIPT_FULL, 2, lambda bf, ss, se: [[("v", 0, b % 3 == 0)] for b in range(16)], W, H)
    if cid == "refine_mid_block_eobr":                                      # tails start at k, after the new value
        pl = _refine_plane(8, 2, 5)
        return _with_refine(pl, SCRIPT_FULL, 2, lambda bf, ss, se: [[("v", 1, False), ("eob", 0, 0)] for _ in range(16)], W, H)
    if cid in ("refine_every_eobr", "refine_eobrun_overshoots_segment"):
        # 256 blocks, restart every 16: segment r opens with EOBr r (r = 0 .. 14), the last with EOBr 4 exactly
        pl = _refine_plane(32, 8, 6)

        def prog(bf, ss, se):
            out = []
            for sg in range(16):
                if cid == "refine_eobrun_overshoots_segment":
                    r, x = 4, 15                                            # 31 blocks claimed in segments of 16
                else:
                    r = sg if sg < 15 else 4
                    x = min((1 << r) - 1, 3)
                n = (1 << r) + x
                seg = [[("eob", r, x)]] + [[] for _ in range(min(n, 16) - 1)]
                if n < 16:
                    seg += [_run_to_end(16 - n)] + [[] for _ in range(15 - n)]
                out += seg
            return out
        return _with_refine(pl, SCRIPT_FULL, 2, prog, 256, 64, restart="16B")
    if cid == "refine_split_bands_ss10":                                    # the 10-63 band, values and tails
        pl = _refine_plane(8, 2, 7)
        return _with_refine(pl, SCRIPT_SPLIT, 4, lambda bf, ss, se: [[("v", 2, b % 2 == 0), ("v", 0, True), ("eob", 0, 0)]
                                                                     for b in range(16)], W, H)
    if cid == "refine_dense_blocks":                                        # every band coefficient nonzero
        pl = _refine_plane(8, 2, 8, dense=True)
        return _with_refine(pl, SCRIPT_FULL, 2, lambda bf, ss, se: [[("zrl",)] if b % 2 else [("eob", 0, 0)] for b in range(16)], W, H)
    if cid in ("refine_size_2", "refine_size_15"):
        size = 2 if cid.endswith("2") else 15
        pl = _refine_plane(8, 2, 9)
        return _with_refine(pl, SCRIPT_FULL, 2, lambda bf, ss, se: [[("v", 0, False), ("eob", 0, 0)] for _ in range(5)]
                            + [[("v", 1, True, size), ("eob", 0, 0)]] + [[("eob", 0, 0)] for _ in range(10)], W, H)
    if cid in ("refine_cut_in_eob_tail", "refine_ends_on_last_correction_bit"):
        for m in range(30, 40):                                             # the last block's tail length sets the bit count
            pl = _refine_plane(8, 2, 10, last_count=m)
            f, car = _with_refine(pl, SCRIPT_FULL, 2, lambda bf, ss, se: [[("v", 0, False)] + _run_to_end(16)]
                                  + [[] for _ in range(15)], W, H)
            toks = refine_tokens(_state(car, 2), 1, 63, [[("v", 0, False)] + _run_to_end(16)] + [[] for _ in range(15)], 0)
            nbits = _token_bits(toks, tables_for([toks]))
            if cid.startswith("refine_ends") and nbits % 8 == 0:
                return f, car
            if cid.startswith("refine_cut") and nbits % 8:
                cut = nbits - nbits % 8                                     # whole bytes, the last block's tail cut
                return replace_scan_bits(car, 2, toks, cut), car
        raise AssertionError("no bit count found")
    if cid in ("refine_empty_segment", "ac_first_empty_segment", "dc_first_empty_segment", "dc_refine_empty_segment",
               "refine_invalid_code", "ac_first_invalid_code", "dc_first_invalid_code"):
        pl = _refine_plane(8, 2, 11)
        script = [((0,), 0, 0, 0, 1), ((0,), 1, 63, 0, 1), ((0,), 0, 0, 1, 0), ((0,), 1, 63, 1, 0)]
        car = carrier(pl, "gray", W, H, script, restart="4B")
        k = {"dc_first": 0, "ac_first": 1, "dc_refine": 2, "refine": 3}[cid.rsplit("_", 2)[0]]
        log = {}
        decode(car, log=log)
        segs = [list(s) for s in log[k]]
        if cid.endswith("empty_segment"):
            segs[2] = []
        else:
            i = next(i for i, t in enumerate(segs[1]) if t[0] == "h")      # where a symbol is due
            segs[1] = segs[1][:i] + [ONES()] + segs[1][i:]
        from mozjpeg_b200 import jpegtran as T
        return splice(car, {k: (write_scan(segs, file_tables(T.parse_source(car), k)), b"")}), car
    if cid in ("ac_first_value_past_se", "ac_first_value_at_se", "ac_first_run_past_63"):
        pl = _refine_plane(8, 2, 12)
        script = [((0,), 0, 0, 0, 0), ((0,), 1, 9, 0, 0), ((0,), 10, 63, 0, 0)]
        car = carrier(pl, "gray", W, H, script)
        k = 2 if cid.endswith("63") else 1
        segs = []
        for b in range(16):
            if cid == "ac_first_run_past_63":                               # at k = 60 a run of 15 lands past 63
                segs += [tok(0xF0), tok(0xF0), tok(0xF0), ac_sym(1, -7), ac_sym(15, 3 + b)]
            elif cid == "ac_first_value_at_se":
                segs += [ac_sym(3, 5), ac_sym(4, -2 - b)]                   # positions 4 and 9 (= Se)
            else:
                segs += [ac_sym(3, 5)] + ([ac_sym(5, 9)] if b == 6 else [eob(0)])   # block 6: position 10 > Se
        return replace_scan(car, k, [segs]), car
    if cid.startswith("ac_first_eobrun_past_end_garbage"):
        rst = cid.endswith("restart")
        pl = _refine_plane(8, 2, 13)
        car = carrier(pl, "gray", W, H, SCRIPT_FULL[:2], restart="8B" if rst else None)
        rng = np.random.default_rng(14)
        nseg = 2 if rst else 1
        segs = []
        for sg in range(nseg):
            toks = [ac_sym(0, 3), ac_sym(2, -1), eob(14, 77)]               # the run claims 16 461 blocks
            for _ in range((2 * S.DEC_SUB_BITS + 300) // 24):               # garbage: random bits, an invalid code inside
                toks.append(B(int(rng.integers(0, 1 << 24)), 24))
            toks.insert(10, ONES())
            segs.append(toks)
        return replace_scan(car, 1, segs), car
    if cid.startswith("dc_refine_8n"):
        plus = cid.endswith("plus_1_blocks")
        wb = 17 if plus else 16
        pl = _refine_plane(wb, 3, 15)
        script = [((0,), 0, 0, 0, 1), ((0,), 1, 63, 0, 0), ((0,), 0, 0, 1, 0)]
        car = carrier(pl, "gray", wb * 8, 24, script, restart=f"{wb}B")
        rng = np.random.default_rng(16)
        segs = [[B(int(rng.integers(0, 1 << 16)), 16)] + ([B(1)] if plus and sg != 1 else []) for sg in range(3)]
        return splice(car, {2: (write_scan(segs, {}), b"")}), car
    if cid == "dc_first_al13_12bit_negative":
        pl = [np.zeros((2, 8, 64), np.int16)]
        script = [((0,), 0, 0, 0, 13)] + [((0,), 0, 0, a, a - 1) for a in range(13, 0, -1)]
        car = carrier(pl, "gray", W, H, script, precision=12)
        diffs = [-1, -1, -1, -1, -1, -1, 2, 7, -15, 3, 1, -2, -1, 0, 4, -6]  # sums reach -6 and +3: -6 << 13 wraps
        return replace_scan(car, 0, [[dc_sym(d) for d in diffs]]), car
    if cid == "second_first_scan":                                          # an AC first scan written twice
        pl = _refine_plane(8, 2, 17)
        car = carrier(pl, "gray", W, H, [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 0)])
        segs = P.segments(car)
        sos = [s for s in segs if s[0] == 0xDA]
        _, a, b = sos[1]
        return car[:b] + car[a:b] + car[b:], car
    raise KeyError(cid)


def _token_bits(toks, tables):
    codes = {key: _codes_of(*t) for key, t in tables.items()}
    return sum((codes[t[1]][t[2]][1] + t[4]) if t[0] == "h" else t[2] for t in toks)


def replace_scan_bits(car, k, toks, nbits):
    """replace_scan of one segment with its bit stream cut to nbits (a whole number of bytes)"""
    tabs = tables_for([toks])
    codes = {key: _codes_of(*t) for key, t in tabs.items()}
    acc, n = 0, 0
    for t in toks:
        if t[0] == "h":
            code, ln = codes[t[1]][t[2]]
            acc, n = (acc << ln | code) << t[4] | t[3], n + ln + t[4]
        else:
            acc, n = acc << t[2] | t[1], n + t[2]
    assert nbits % 8 == 0 and nbits < n
    data = (acc >> (n - nbits)).to_bytes(nbits // 8, "big").replace(b"\xff", b"\xff\x00")
    return splice(car, {k: (data, _dht(tabs))})


# ------------------------------------------------------------------------------------------------ damaged files
def _std_gray(W, H, seed, restart=None):
    pl = S.planes("mixed", "gray", W, H, 8, seed)
    return S.encode(pl, "gray", W, H, scans="prog", restart=restart)


MUTANT_SOURCES = ["gray_std", "gray_std_rst1b", "ragged_420_rst_rows", "422_split_script", "gray12_al13", "default_profile",
                  "corrections"]


def mutant_source(sid) -> bytes:
    if sid == "gray_std":
        return _std_gray(40, 32, 1)
    if sid == "gray_std_rst1b":
        return _std_gray(40, 24, 2, "1B")
    if sid == "ragged_420_rst_rows":                   # interleaved DC first at Al 1, a DC refinement with dummy blocks
        pl = S.planes("mixed", "2x2", 41, 27, 8, 3)
        return S.encode(pl, "2x2", 41, 27, scans="prog", restart="1")
    if sid == "422_split_script":
        for seed in range(4, 40):
            pl = S.planes("mixed", "2x1", 40, 24, 8, seed)
            f = S.encode(pl, "2x1", 40, 24, scans="script", seed=seed)
            from mozjpeg_b200 import jpegtran as T
            info = T.parse_source(f)
            if any(0 < sc.Ss and sc.Se < 63 and sc.Ah for sc in info.scans[:info.num_scans]):
                return f
        raise AssertionError("no split-band script")
    if sid == "gray12_al13":
        pl = S.planes("mixed", "gray", 32, 24, 12, 5)
        return S.encode(pl, "gray", 32, 24, precision=12, scans="script", seed=5)
    if sid == "default_profile":
        return P.source(("default_small", 48, 32, 6, ["-quality", "75"]))
    if sid == "corrections":
        return P.extra_source("carrier_corrections")
    raise KeyError(sid)


def scan_mutants(good: bytes, k: int, n: int, seed: int):
    """n seeded damaged copies of `good` with scan k's entropy-coded data damaged: bit flips, byte deletions and
    insertions, RSTn renumbering and truncations (the file cut inside the scan and EOI appended, so later scans go).
    A mutant that creates or removes a marker (truncation and RSTn renumbering aside) is dropped.  [(kind, bytes)]"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(good)
    sc = info.scans[k]
    lo, hi = sc.data_offset, sc.data_offset + sc.data_size
    want = S._marker_kinds(good, lo)
    rsts = [m.start(1) for m in re.finditer(rb"\xff([\xd0-\xd7])", good[lo:hi])]
    rng = np.random.default_rng(seed)
    kinds = ["flip", "flip", "flip", "delete", "insert", "truncate"] + (["renumber"] if rsts else [])
    out, tries = [], 0
    while len(out) < n and tries < 50 * n:
        tries += 1
        kd = kinds[int(rng.integers(0, len(kinds)))]
        d = bytearray(good)
        if kd == "flip":
            p = int(rng.integers(lo, hi))
            d[p] ^= 1 << int(rng.integers(0, 8))
        elif kd == "delete":
            del d[int(rng.integers(lo, hi))]
        elif kd == "insert":
            d.insert(int(rng.integers(lo, hi + 1)), int(rng.integers(0, 256)))
        elif kd == "renumber":
            p = lo + rsts[int(rng.integers(0, len(rsts)))]
            d[p] = 0xD0 + (d[p] - 0xD0 + int(rng.integers(1, 8))) % 8
        else:
            d = d[:int(rng.integers(lo, hi))] + bytearray(b"\xff\xd9")
        d = bytes(d)
        if kd != "truncate" and S._marker_kinds(d, lo) != want:
            continue
        out.append((kd, d))
    return out


MUTANTS_PER_SCAN = 3


def all_mutants(sid):
    """[(scan kind, scan, kind of damage, bytes)] of a source: MUTANTS_PER_SCAN per scan"""
    from mozjpeg_b200 import jpegtran as T
    good = mutant_source(sid)
    info = T.parse_source(good)
    out = []
    for k in range(info.num_scans):
        for kd, m in scan_mutants(good, k, MUTANTS_PER_SCAN, seed=1000 * len(sid) + k):
            out.append((kind(info.scans[k]), k, kd, m))
    return out
