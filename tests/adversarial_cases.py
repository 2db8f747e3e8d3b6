"""Constructed inputs that drive the encoder into its content-dependent edge cases, and plain references to measure
that they do.  numpy only, no GPU.

Smooth-plus-noise test images leave it to chance whether the exactness rules of the quantizers, the trellis and the
entropy coder are ever exercised.  Each family below forces one of them:

* pixel families (8-bit, some 12-bit): flat-block level ladders under swept quantization tables, blocks built from
  chosen DCT basis functions (every non-zero count 0..63, runs across zigzag position 31/32), and screen-like content
  (hard edges, checkerboards, one-level gradients, repeated blocks, alternating 0/255 blocks, noise next to flat blocks);
* coefficient families (natural-order int16 planes, jpeg_write_coefficients input): Fibonacci and equal symbol
  frequencies, a single symbol, every symbol the precision allows, magnitudes at the coefficient limit, progressive
  images of 32767..65536 mostly empty blocks, refinement blocks whose correction bits add up to the 937-bit flush, and
  streams that are mostly 0xFF bytes.

The references are written from the JPEG specification and the reference's documented rules, independently of the
C restatement in oracle/: symbol histograms of a sequential scan, jpeg_gen_optimal_table (jchuff.c:947-1106), per-block
symbol counts and the EOBRUN runs of progressive AC scans (jcphuff.c encode_mcu_AC_first / encode_mcu_AC_refine).
"""
import numpy as np

# zigzag position -> natural index
ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
               21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
               61, 54, 47, 55, 62, 63])


def nbits(v):
    """Bits of |v| (0 for 0), elementwise."""
    a = np.abs(np.asarray(v, dtype=np.int64))
    out = np.zeros(a.shape, dtype=np.int64)
    while (a > 0).any():
        out += a > 0
        a >>= 1
    return out


def _blocks_to_image(blocks, wb):
    """(n, 8, 8) blocks -> one image wb blocks wide (the last row padded with copies of the last block)."""
    n = len(blocks)
    hb = -(-n // wb)
    blocks = np.concatenate([blocks, np.repeat(blocks[-1:], hb * wb - n, 0)])
    return blocks.reshape(hb, wb, 8, 8).transpose(0, 2, 1, 3).reshape(hb * 8, wb * 8)


# ---------------------------------------------------------------------------------------------------------------------
# pixel families
# ---------------------------------------------------------------------------------------------------------------------
def flat_ladder(precision=8):
    """Gray image whose blocks are flat, one level each: every level 0..255 at 8 bits; at 12 bits every 16th level
    plus 2047, 2048 and 4095.  Swept against quantization tables this covers the whole DC quantizer."""
    if precision == 8:
        levels = np.arange(256)
    else:
        levels = np.unique(np.concatenate([np.arange(0, 4096, 16), [1, 2047, 2048, 2049, 4094, 4095]]))
    blocks = np.repeat(levels[:, None, None], 64, 1).reshape(-1, 8, 8)
    return _blocks_to_image(blocks, 16).astype(np.uint8 if precision == 8 else np.uint16)


def flat_tables(values, force_baseline=True):
    """(len(values), 4, 64) quantization tables: set i has every DC and AC entry of every slot equal to values[i]."""
    v = np.asarray(values, dtype=np.int64)
    if force_baseline:
        v = np.clip(v, 1, 255)
    return np.repeat(v[:, None], 4 * 64, 1).reshape(len(v), 4, 64).astype(np.uint16)


def _idct_matrix():
    """Orthonormal 8-point DCT-II basis: the JPEG FDCT is C @ x @ C.T (jcdctmgr's outputs are 8x this)."""
    k = np.arange(8)
    c = np.sqrt(2 / 8) * np.cos((2 * k[None, :] + 1) * k[:, None] * np.pi / 16)
    c[0] /= np.sqrt(2)
    return c


def basis_block(coefs_zz, q):
    """Pixels (8x8, uint8) whose DCT is coefs_zz (64 values in zigzag order, in units of the quantizer step q) around
    mid-grey, rounded and clipped."""
    nat = np.zeros(64)
    nat[ZZ] = np.asarray(coefs_zz, dtype=np.float64) * q
    c = _idct_matrix()
    pix = c.T @ nat.reshape(8, 8) @ c + 128.0
    return np.clip(np.rint(pix), 0, 255).astype(np.uint8)


def basis_patterns(seed=0):
    """Zigzag-ordered AC patterns (in quantizer steps): every non-zero count 0..63 (values +-1 and +-2, random
    positions), runs of 15, 16, 17, 31, 32 and 47 zeros across position 31/32, a lone value at 63, and half-way
    amplitudes (k + 1/2) that put the raw coefficient on a rounding tie."""
    rng = np.random.default_rng(seed)
    pats = []
    for n in range(64):
        for rep in range(2):
            z = np.zeros(64)
            pos = rng.choice(np.arange(1, 64), n, replace=False)
            z[pos] = rng.choice([-2, -1, 1, 2], n) if rep else rng.choice([-1, 1], n)
            pats.append(z)
    for run in (15, 16, 17, 31, 32, 47):
        for a in sorted({max(1, 31 - run), max(1, 31 - run // 2), 30, 31}):
            b = a + run + 1
            if b <= 63:
                z = np.zeros(64); z[a] = 1; z[b] = -1
                pats.append(z)
                z = z.copy(); z[1:a] = 1                        # dense head, then the run across 31/32
                pats.append(z)
    z = np.zeros(64); z[63] = 1; pats.append(z)
    z = np.zeros(64); z[63] = -3; z[1] = 2; pats.append(z)
    for k in range(4):
        z = np.zeros(64); z[1:9] = k + 0.5; z[40:44] = -(k + 0.5); pats.append(z)
    return pats


def basis_image(q=16, seed=0):
    """Gray image of basis_patterns blocks at quantizer step q, 16 blocks wide."""
    return _blocks_to_image(np.stack([basis_block(z, q) for z in basis_patterns(seed)]), 16)


def screen_images(seed=0):
    """name -> 8-bit RGB screen-like image (128x128 unless stated)."""
    rng = np.random.default_rng(seed)
    h = w = 128
    yy, xx = np.indices((h, w))
    out = {}
    e = np.zeros((h, w), np.uint8); e[:, 64:] = 255; e[64:, :] ^= 0xFF
    out["edges_aligned"] = e
    e = np.zeros((h, w), np.uint8); e[:, 63:] = 255; e[65:, :] = 40; e[:, 9:10] = 200
    out["edges_off_by_one"] = e
    for per in (1, 2, 4, 8, 16):
        for ph in range(0, 2 * per, max(1, per // 2)):
            out["checker_p%d_ph%d" % (per, ph)] = ((((yy + ph) // per + (xx + ph) // per) % 2) * 255).astype(np.uint8)
    out["gradient_h"] = (xx * 2 + yy // 64).astype(np.uint8)
    out["gradient_v"] = (yy * 2 + xx // 64).astype(np.uint8)
    tile = rng.integers(0, 256, (8, 8), dtype=np.uint8)
    out["repeated_block"] = np.tile(tile, (h // 8, w // 8))
    out["alternating_0_255"] = ((((yy // 8) + (xx // 8)) % 2) * 255).astype(np.uint8)
    # noise whose amplitude grows block by block (a few non-zero values up to all 63 at q100), next to flat blocks
    amp = np.repeat(np.repeat(np.geomspace(0.3, 40, (h // 8) * (w // 8)).reshape(h // 8, w // 8), 8, 0), 8, 1)
    nz = np.clip(np.rint(128 + rng.standard_normal((h, w)) * amp), 0, 255)
    flat = ((yy // 8 + xx // 16) % 3 == 0)
    out["noise_and_flat"] = np.where(flat, 77, nz).astype(np.uint8)
    rgb = {}
    for k, g in out.items():
        # three related planes so that chroma carries edges too (and not just a grey copy)
        rgb[k] = np.stack([g, np.roll(g, 3, 1), 255 - g], axis=2)
    return rgb


def gradient12():
    """12-bit gray image stepping one level per pixel through 0..4095 (64x64), and its mirror."""
    v = np.arange(4096, dtype=np.uint16).reshape(64, 64)
    return np.concatenate([v, v[::-1, ::-1]], axis=1)


# ---------------------------------------------------------------------------------------------------------------------
# coefficient families: (hib, wib, 64) int16 planes in natural order
# ---------------------------------------------------------------------------------------------------------------------
def _value_of_size(s, sign=1, ones=False):
    """A coefficient of size s: 2^(s-1) (value bits 10..0), or 2^s - 1 (value bits all ones) with ones=True."""
    v = (1 << s) - 1 if ones else 1 << (s - 1)
    return sign * v


def pack_ac_symbols(symbols, wb=32, dc=None):
    """Blocks (natural order) that together contain exactly the given AC (run, size) symbols, each block filled in
    zigzag order until the next symbol does not fit.  Returns the (hib, wib, 64) plane."""
    blocks = []
    cur = np.zeros(64, np.int16); pos = 1
    for i, (r, s) in enumerate(symbols):
        if pos + r > 63:
            blocks.append(cur); cur = np.zeros(64, np.int16); pos = 1
        cur[ZZ[pos + r]] = _value_of_size(s, 1 if i % 2 else -1)
        pos += r + 1
    blocks.append(cur)
    b = np.stack(blocks)
    n = len(b)
    hb = -(-n // wb)
    b = np.concatenate([b, np.zeros((hb * wb - n, 64), np.int16)])
    if dc is not None:
        b[:, 0] = dc_walk(dc, len(b))
    return b.reshape(hb, wb, 64)


def dc_walk(sizes, n):
    """n DC values whose successive differences have the given sizes (cycled), staying inside +-1023."""
    sizes = list(sizes)
    out = np.zeros(n, np.int64)
    cur = 0
    for i in range(n):
        s = sizes[i % len(sizes)]
        d = 0 if s == 0 else (1 << (s - 1))
        cur = cur - d if cur > 0 else cur + d
        out[i] = cur
    return out.astype(np.int16)


def fib_symbols(max_size=10, count=21):
    """AC symbols with Fibonacci frequencies 1, 2, 3, 5, ... (next to the reserved symbol's 1 this makes a chain, one
    level per symbol): the unlimited Huffman code lengths reach the 20s, which the 16-bit length limit (Annex K.2)
    has to fold back."""
    syms = [(r, s) for r in (0, 1, 2, 3) for s in range(1, max_size + 1)][:count]
    f = [1, 2]
    while len(f) < count:
        f.append(f[-1] + f[-2])
    out = []
    for (r, s), k in zip(syms, f):
        out += [(r, s)] * k
    rng = np.random.default_rng(1)
    rng.shuffle(out)
    return out


def equal_symbols(max_size=10, each=7):
    """Every (run 0..3, size) symbol exactly ``each`` times: Huffman merges decided by the tie rule alone."""
    out = [(r, s) for r in range(4) for s in range(1, max_size + 1)] * each
    return out


def all_symbols(max_size):
    """Every AC symbol with a size up to max_size, runs 0..15, each twice, plus long runs that need ZRL."""
    out = [(r, s) for r in range(16) for s in range(1, max_size + 1)] * 2
    return out + [(15, 1), (15, max_size), (20, 1), (40, max_size)] * 3       # runs of 16 and more need ZRL


def coef_families(precision=8):
    """name -> (planes list for one gray image, description).  max AC size = precision + 2, DC difference size
    precision + 3."""
    mx = precision + 2
    fam = {}
    fam["fib"] = pack_ac_symbols(fib_symbols(mx), dc=[0, 1, 1, 2, 3, 5, 8, 11][: mx + 1])
    f = [1, 2]
    while len(f) < mx + 2:
        f.append(f[-1] + f[-2])
    sizes = np.random.default_rng(2).permutation(np.repeat(np.arange(mx + 2), f[::-1]))     # every DC size, Fibonacci counts
    n = -(-len(sizes) // 32) * 32
    dcp = np.zeros((n, 64), np.int16)
    dcp[:, 0] = dc_walk(np.concatenate([sizes, np.zeros(n - len(sizes), np.int64)]), n)
    fam["fib_dc"] = dcp.reshape(-1, 32, 64)
    fam["equal"] = pack_ac_symbols(equal_symbols(mx), dc=list(range(mx + 2)))
    fam["single_symbol"] = np.zeros((4, 8, 64), np.int16)
    fam["all_symbols"] = pack_ac_symbols(all_symbols(mx), dc=list(range(min(mx + 2, 12))))
    edge = np.zeros((2, 8, 64), np.int16)
    edge[0, :, 1] = (1 << mx) - 1; edge[0, :, 63] = -((1 << mx) - 1); edge[1, ::2, 0] = 1023; edge[1, 1::2, 0] = -1023
    fam["max_magnitude"] = edge
    return {k: [v.astype(np.int16)] for k, v in fam.items()}


def out_of_range_plane(precision=8):
    """One AC value of size max_coef_bits + 1: the reference stops with JERR_BAD_DCT_COEF."""
    a = np.zeros((2, 2, 64), np.int16)
    a[1, 1, 5] = 1 << (precision + 2)
    return [a]


def eobrun_plane(nblocks):
    """Gray planes of nblocks blocks (32767, 32768, 65535, 65536), empty except isolated blocks next to multiples of
    256 (the progressive kernels' tile) and of 0x7FFF, with gaps of exactly 0x7FFF empty blocks (the whole 32767-block
    image is one)."""
    shapes = {32767: (151, 217), 32768: (128, 256), 65535: (255, 257), 65536: (256, 256)}
    marks = {32767: [], 32768: [0x7FFF], 65535: [255, 256, 257, 257 + 0x8000, 65534],
             65536: [0, 256, 511, 512, 512 + 0x8000, 65535]}[nblocks]
    hb, wb = shapes[nblocks]
    b = np.zeros((hb * wb, 64), np.int16)
    for i, m in enumerate(marks):
        b[m, ZZ[[1, 2, 5, 30, 33]]] = [1, 3, -2, 1, -5 + i % 3]
        b[m, 0] = 4
    return [b.reshape(hb, wb, 64)]


def correction_plane(wb=32, rows=8):
    """Gray plane for an AC refinement (Ah=1, Al=0) scan: no value becomes newly non-zero, so every block joins the
    EOB run and adds its correction bits (|value| >= 2 at 62 or fewer positions).  Fifteen blocks of 62 bits and one
    of 8 sum to 938, the first total past the 937-bit flush; others sum to exactly 937."""
    counts = []
    while len(counts) < wb * rows:
        counts += [62] * 15 + [8] + [62] * 15 + [7] + [1] * 3 + [61]
    counts = counts[: wb * rows]
    b = np.zeros((wb * rows, 64), np.int16)
    for i, c in enumerate(counts):
        pos = np.arange(1, 1 + c)
        b[i, ZZ[pos]] = np.where(pos % 3 == 0, -3, 2)
    return [b.reshape(rows, wb, 64)]


REFINE_SCANS = "0: 0-0, 0, 0;\n0: 1-63, 0, 1;\n0: 1-63, 1, 0;\n"


def ff_plane(wb=128, hb=96):
    """8-bit gray plane for the standard tables (-revert): runs of 15 zeros then 1023, four per block ending at
    position 63 (no EOB), DC difference 0.  Codes 1111111111111110 / ...101 followed by ten one-bits make the unstuffed
    stream mostly 0xFF bytes."""
    b = np.zeros((hb * wb, 64), np.int16)
    b[:, ZZ[[16, 32, 48, 63]]] = 1023
    return [b.reshape(hb, wb, 64)]


# ---------------------------------------------------------------------------------------------------------------------
# plain references
# ---------------------------------------------------------------------------------------------------------------------
def block_ac_symbols(zz):
    """The AC symbols encode_one_block (jchuff.c) emits for one block given in zigzag order: (run << 4 | size) for each
    non-zero value, 0xF0 for every 16 zeros before it, 0x00 (EOB) unless position 63 is non-zero."""
    out = []
    r = 0
    for k in range(1, 64):
        v = int(zz[k])
        if v == 0:
            r += 1
            continue
        while r > 15:
            out.append(0xF0); r -= 16
        out.append((r << 4) | int(nbits(v)))
        r = 0
    if r > 0:
        out.append(0x00)
    return out


def seq_histograms(planes_nat):
    """Per component: (DC histogram [17], AC histogram [257]) of a sequential scan over the (hib, wib, 64) natural-order
    planes, blocks in raster order (no restarts)."""
    res = []
    for pl in planes_nat:
        zz = pl.reshape(-1, 64)[:, ZZ].astype(np.int64)
        dc = np.zeros(17, np.int64); ac = np.zeros(257, np.int64)
        diffs = np.diff(np.concatenate([[0], zz[:, 0]]))
        np.add.at(dc, nbits(diffs), 1)
        for blk in zz:
            for s in block_ac_symbols(blk):
                ac[s] += 1
        res.append((dc, ac))
    return res


def symbols_per_block(plane_nat):
    """Number of AC symbols (values, ZRLs and EOB) of every block of a natural-order plane."""
    zz = plane_nat.reshape(-1, 64)[:, ZZ]
    return np.array([len(block_ac_symbols(b)) for b in zz])


def nonzero_ac_counts(plane_nat):
    return (plane_nat.reshape(-1, 64)[:, 1:] != 0).sum(1)


def code_lengths(freq):
    """Unlimited Huffman code lengths of jpeg_gen_optimal_table's merge loop over freq[0..255] plus the reserved
    symbol 256 (frequency 1): the two smallest frequencies merge, the larger symbol index winning ties."""
    f = [int(x) for x in freq[:256]] + [0] * (256 - len(freq[:256])) + [1]
    codesize = [0] * 257
    others = [-1] * 257
    while True:
        c1 = c2 = -1
        for i in range(257):
            if f[i] and (c1 < 0 or f[i] <= f[c1]):
                c1 = i
        for i in range(257):
            if f[i] and i != c1 and (c2 < 0 or f[i] <= f[c2]):
                c2 = i
        if c2 < 0:
            break
        f[c1] += f[c2]; f[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]; codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]; codesize[c2] += 1
    return codesize


def gen_optimal_table(freq):
    """jpeg_gen_optimal_table (jchuff.c:947-1106, ITU T.81 Annex K.2): (bits[0..16], huffval) of the optimal table,
    code lengths limited to 16 and the all-ones code of the reserved symbol removed.  Also returns the largest
    unlimited code length."""
    codesize = code_lengths(freq)
    bits = [0] * 33
    for i in range(257):
        if codesize[i]:
            bits[codesize[i]] += 1
    longest = max(codesize)
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2; bits[i - 1] += 1; bits[j + 1] += 2; bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    huffval = [s for n in range(1, 33) for s in range(256) if codesize[s] == n]
    return tuple(bits[:17]), tuple(huffval), longest


def eobruns(plane_nat, Ss, Se, Ah, Al):
    """Progressive AC scan of one component (jcphuff.c encode_mcu_AC_first when Ah == 0, encode_mcu_AC_refine
    otherwise), no restarts: the EOBRUN symbols it emits, as (run length, correction bits flushed with it,
    reason) with reason 'max' (the run reached 0x7FFF), 'be' (more than 937 buffered correction bits) or 'data'
    (a value or the end of the scan ended it)."""
    zz = np.abs(plane_nat.reshape(-1, 64)[:, ZZ].astype(np.int64)) >> Al
    out = []
    E = BE = 0

    def emit(reason):
        nonlocal E, BE
        if E:
            out.append((E, BE, reason))
        E = BE = 0

    for blk in zz:
        r = 0
        if Ah == 0:
            for k in range(Ss, Se + 1):
                if blk[k] == 0:
                    r += 1
                    continue
                emit("data")
                r = 0
            if r > 0:
                E += 1
                if E == 0x7FFF:
                    emit("max")
        else:
            last1 = max([k for k in range(Ss, Se + 1) if blk[k] == 1], default=-1)
            br = 0
            for k in range(Ss, Se + 1):
                t = blk[k]
                if t == 0:
                    r += 1
                    continue
                while r > 15 and k <= last1:
                    emit("data"); r -= 16; br = 0
                if t > 1:
                    br += 1
                    continue
                emit("data")
                br = 0; r = 0
            if r > 0 or br > 0:
                E += 1; BE += br
                if E == 0x7FFF:
                    emit("max")
                elif BE > 937:
                    emit("be")
    emit("data")
    return out


def scan_segments(jpeg):
    """The entropy-coded bytes of every scan, unstuffed (FF 00 -> FF, restart markers dropped)."""
    out = []
    pos = 2
    while pos + 4 <= len(jpeg):
        m = jpeg[pos + 1]
        ln = (jpeg[pos + 2] << 8) | jpeg[pos + 3]
        if m != 0xDA:
            pos += 2 + ln
            continue
        pos += 2 + ln
        seg = bytearray()
        while pos < len(jpeg):
            b = jpeg[pos]
            if b == 0xFF:
                n = jpeg[pos + 1]
                if n == 0x00:
                    seg.append(0xFF); pos += 2; continue
                if 0xD0 <= n <= 0xD7:
                    pos += 2; continue
                break
            seg.append(b); pos += 1
        out.append(bytes(seg))
    return out


def max_ff_share(jpeg, tile=4096):
    """Largest share of 0xFF bytes in any whole 4096-byte tile of any unstuffed scan, and the number of tiles."""
    best, tiles = 0.0, 0
    for seg in scan_segments(jpeg):
        a = np.frombuffer(seg, np.uint8)
        for t in range(len(a) // tile):
            tiles += 1
            best = max(best, float((a[t * tile:(t + 1) * tile] == 0xFF).mean()))
    return best, tiles
