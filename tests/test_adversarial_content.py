"""Constructed content (tests/adversarial_cases.py) that reaches the content-dependent exactness rules of the encoder:
the DC quantizer over every level and table value, exact rounding ties of the float quantizer and of the trellis,
every non-zero count a block can have, zero runs across zigzag position 31/32, symbol records of 15, 16, 31, 32 and
more entries, Huffman code lengths past 16, EOB runs cut at 0x7FFF and at 937 buffered correction bits, and entropy
streams that are mostly 0xFF.

CPU tests: every family reaches its edge (measured with the plain references or the restatement's taps), and the
restatement (oracle/jpeg_oracle.c) writes the unmodified reference's bytes on it (skipped without oracle/_ref).
GPU tests: the device writes the restatement's bytes on the same inputs, across the DCTs, sampling layouts, ragged
sizes, trellis modes, progressive scripts, the scan search, restarts and chunked batches; a mismatch names the first
stage (raw / plain / final coefficients, trellis-phase or per-scan Huffman tables) that differs."""
import os
import tempfile

import numpy as np
import pytest

import adversarial_cases as AC

# the per-image tables of the ladders: the full baseline range on the device, a spread of it against the reference
Q_BASELINE = list(range(1, 256))
Q_BASELINE_REF = [1, 2, 3, 7, 16, 31, 100, 128, 255]
Q_WIDE = [1, 2, 16, 255, 256, 1000, 4095, 16383, 16384, 32767]
TWELVE = ["-precision", "12", "-notrellis", "-noovershoot"]


def _need_ref(tool=None):
    from oracle import oracle as O
    if not O.ref_available() or (tool and not os.path.exists(os.path.join(O.REF_DIR, tool))):
        pytest.skip("oracle/_ref not built")


def _params(sw, img):
    import mozjpeg_b200 as mj
    nc = 1 if img.ndim == 2 else img.shape[2]
    return mj.params_from_switches(sw, img.shape[1], img.shape[0], nc)


def _with_tables(p, t):
    c = p.copy()
    np.ctypeslib.as_array(c.quant_tbl)[:] = t
    return c


def _tables_file(d, t):
    path = os.path.join(d, "q.txt")
    with open(path, "w") as f:
        for _ in range(4):
            f.write(" ".join(str(int(v)) for v in t.reshape(-1)[:64]) + "\n")      # flat: natural and zigzag order agree
    return path


def _ref_pixels(img, sw, precision=8):
    """The reference cjpeg on an in-memory image; 12-bit samples go through a maxval-4095 PGM/PPM."""
    from oracle import oracle as O
    if precision == 8:
        return O._ref_cjpeg_pixels(img, sw)
    gray = img.ndim == 2
    with tempfile.NamedTemporaryFile(suffix=".pgm" if gray else ".ppm") as f:
        f.write(b"%s\n%d %d\n4095\n" % (b"P5" if gray else b"P6", img.shape[1], img.shape[0]))
        f.write(np.ascontiguousarray(img, dtype=">u2").tobytes()); f.flush()
        return O.ref_cjpeg(f.name, sw)


def _dht_tables(jpeg):
    """(class, id) -> bits[1..16] of every DHT segment of a file."""
    out, pos = {}, 2
    while pos + 4 <= len(jpeg) and jpeg[pos + 1] != 0xDA:
        ln = (jpeg[pos + 2] << 8) | jpeg[pos + 3]
        if jpeg[pos + 1] == 0xC4:
            q = pos + 4
            while q < pos + 2 + ln:
                bits = tuple(jpeg[q + 1:q + 17])
                out.setdefault((jpeg[q] >> 4, jpeg[q] & 15), []).append(bits)
                q += 17 + sum(bits)
        pos += 2 + ln
    return out


# ---------------------------------------------------------------------------------------------------------------------
# coefficient carriers: the restatement writes a plain file holding the crafted planes; jpegtran re-encodes it
# ---------------------------------------------------------------------------------------------------------------------
def _carrier(planes, precision=8):
    from oracle import oracle as O
    hib, wib = planes[0].shape[:2]
    sw = (["-precision", "12"] if precision == 12 else []) + ["-revert"]
    import mozjpeg_b200 as mj
    p = mj.params_from_switches(sw, wib * 8, hib * 8, 1)
    return O.oracle_encode_coefs(p, planes)


def _transcode_params(src, tsw, scans=None):
    """(params, prefer_smallest) of ``jpegtran <tsw> [-scans file]``: the scan script is read after the switches'
    progression, as jpegtran does, and turns prefer_smallest off."""
    from mozjpeg_b200 import jpegtran as T
    from mozjpeg_b200.cjpeg import _read_scan_script
    p, prefer = T.params_for_transcode(T.parse_header(src), tsw)
    if scans:
        _read_scan_script(p, scans)
        prefer = False
    return p, prefer


def _oracle_transcode(src, planes, tsw, scans=None):
    from mozjpeg_b200 import _abi as A
    from oracle import oracle as O
    p, prefer = _transcode_params(src, tsw, scans)
    out = O.oracle_encode_coefs(p, planes)
    if prefer and p.compress_profile == A.PROFILE_MAX_COMPRESSION and len(src) < len(out):
        out = src
    return out


def _scans_file(d):
    path = os.path.join(d, "refine.txt")
    with open(path, "w") as f:
        f.write(AC.REFINE_SCANS)
    return path


TRAN = [[], ["-revert"], ["-revert", "-optimize"], ["-progressive"], ["-revert", "-optimize", "-restart", "1"]]


def _coef_cases():
    """(id, planes, precision, jpegtran switches, use the refinement script)."""
    cases = []
    for prec in (8, 12):
        for name, planes in AC.coef_families(prec).items():
            for tsw in TRAN:
                cases.append(("%s%d:%s" % (name, prec, "_".join(s.lstrip("-") for s in tsw) or "default"), planes, prec, tsw, False))
    for n in (32767, 32768, 65535, 65536):
        cases.append(("eobrun%d:scans" % n, AC.eobrun_plane(n), 8, [], True))
    cases.append(("eobrun65536:progressive", AC.eobrun_plane(65536), 8, ["-progressive"], False))
    cases.append(("correction:scans", AC.correction_plane(), 8, [], True))
    cases.append(("correction:revert_scans", AC.correction_plane(), 8, ["-revert"], True))
    cases.append(("ff:revert", AC.ff_plane(), 8, ["-revert"], False))
    cases.append(("ff:revert_restart", AC.ff_plane(), 8, ["-revert", "-restart", "1"], False))
    return cases


COEF_CASES = _coef_cases()


# ---------------------------------------------------------------------------------------------------------------------
# CPU: every family reaches its edge
# ---------------------------------------------------------------------------------------------------------------------
def test_basis_blocks_reach_every_nonzero_count_and_run(built):
    from oracle import oracle as O
    img = AC.basis_image()
    p = _with_tables(_params(["-baseline"], img), AC.flat_tables([16])[0])
    d = O.oracle_encode(p, img, want_debug=True).dbg
    plain = d["plain"][0][:d["hib"][0], :d["wib"][0]]
    assert set(AC.nonzero_ac_counts(plain)) == set(range(64))
    runs = set()
    for b in plain.reshape(-1, 64)[:, AC.ZZ]:
        nz = [0] + [k for k in range(1, 64) if b[k]]
        runs |= {bb - a - 1 for a, bb in zip(nz, nz[1:]) if a < 32 <= bb}
    assert {15, 16, 17, 31, 32, 47} <= runs
    assert any(b[AC.ZZ[63]] and not b[AC.ZZ[1:63]].any() for b in plain.reshape(-1, 64))


def test_noise_and_flat_reaches_every_symbol_record_class(built):
    """Trellis output of q95 noise next to flat blocks: symbol records of 15 / 16 entries (the split record), 31 / 32
    (the overflow at 31 slots) and more, next to one-entry records."""
    from oracle import oracle as O
    img = AC.screen_images()["noise_and_flat"]
    p = _params(["-baseline", "-quality", "95", "-sample", "1x1"], img)
    d = O.oracle_encode(p, img, want_debug=True).dbg
    counts = set()
    for ci in range(3):
        counts |= set(AC.symbols_per_block(d["final"][ci][:d["hib"][ci], :d["wib"][ci]]))
    assert {1, 15, 16, 31, 32} <= counts and max(counts) > 32
    nz = AC.nonzero_ac_counts(d["plain"][0])
    assert nz.min() <= 8 and ((nz >= 9) & (nz <= 15)).any() and ((nz >= 16) & (nz <= 32)).any() and nz.max() > 32


def test_flat_ladder_reaches_exact_dc_halves(built):
    """Odd offsets from 128 under Q = 16: the raw DC is an exact half-step, and the float quantizer's +16384.5 rounds
    it up where the integer quantizer rounds away from zero."""
    from oracle import oracle as O
    img = AC.flat_ladder()
    for dct in ("int", "float"):
        p = _with_tables(_params(["-baseline", "-dct", dct], img), AC.flat_tables([16])[0])
        d = O.oracle_encode(p, img, want_debug=True).dbg
        raw = d["raw"][0][..., 0].astype(np.int64)
        assert (np.abs(raw) % 128 == 64).sum() >= 128
    lv = np.arange(256)
    assert (d["plain"][0][..., 0].reshape(-1)[:256] == np.floor((lv - 128) / 2 + 0.5)).all()


def test_twelve_bit_ladder_reaches_the_quantizer_bound():
    """|x| + d/2 < 2^18 is where the multiply-shift quantizers stay exact: a black 12-bit block under Q = 32767 sits
    just below it."""
    img = AC.flat_ladder(12)
    raw = 64 * (int(img.min()) - 2048)
    d = 8 * max(Q_WIDE)
    assert img.min() == 0 and img.max() == 4095 and 2 ** 18 - 8 <= abs(raw) + d // 2 < 2 ** 18


def test_fibonacci_frequencies_need_the_length_limit(built):
    from oracle import oracle as O
    planes = AC.coef_families(8)["fib"]
    _, ac = AC.seq_histograms(planes)[0]
    bits, _, longest = AC.gen_optimal_table(ac)
    assert longest > 16 and bits[16] > 0
    out = _oracle_transcode(_carrier(planes), planes, ["-revert", "-optimize"])
    assert any(b[15] > 0 for b in _dht_tables(out)[(1, 0)])


def test_equal_and_single_symbol_histograms():
    _, ac = AC.seq_histograms(AC.coef_families(8)["equal"])[0]
    vals = ac[np.nonzero(ac)[0]]
    assert (vals == 7).sum() >= 40
    _, ac = AC.seq_histograms(AC.coef_families(8)["single_symbol"])[0]
    assert np.count_nonzero(ac) == 1


def test_every_symbol_the_precision_allows():
    for prec in (8, 12):
        dc, ac = AC.seq_histograms(AC.coef_families(prec)["all_symbols"])[0]
        assert all(ac[(r << 4) | s] for r in range(16) for s in range(1, prec + 3)) and ac[0xF0]
        dc, _ = AC.seq_histograms(AC.coef_families(prec)["fib_dc"])[0]
        assert (dc[:prec + 4] > 0).all()


def test_progressive_runs_reach_0x7fff_and_the_937_bit_flush():
    for n in (32767, 32768, 65535, 65536):
        runs = AC.eobruns(AC.eobrun_plane(n)[0], 1, 63, 1, 0) + AC.eobruns(AC.eobrun_plane(n)[0], 1, 63, 0, 1)
        assert any(r[2] == "max" and r[0] == 0x7FFF for r in runs), n
    runs = AC.eobruns(AC.correction_plane()[0], 1, 63, 1, 0)
    be = [r[1] for r in runs if r[2] == "be"]
    assert 938 in be and all(b > 937 for b in be)
    assert all(r[1] <= 937 for r in runs if r[2] != "be")


def test_ff_stream_is_mostly_ff(built):
    planes = AC.ff_plane()
    for tsw in (["-revert"], ["-revert", "-restart", "1"]):
        share, tiles = AC.max_ff_share(_oracle_transcode(_carrier(planes), planes, tsw))
        assert share >= 0.5 and tiles > 32, (tsw, share, tiles)


def test_gen_optimal_table_matches_the_restatement(built):
    import ctypes as C
    from mozjpeg_b200 import _abi as A
    from oracle import oracle as O
    for prec in (8, 12):
        for name, planes in AC.coef_families(prec).items():
            for hist in AC.seq_histograms(planes)[0]:
                bits, huffval, _ = AC.gen_optimal_table(hist)
                f = (C.c_long * 257)(*[int(x) for x in hist] + [0] * (257 - len(hist)))
                t = A.HuffTbl()
                O.orc().orc_gen_optimal_table(f, C.byref(t))
                assert O._huff_to_py(t) == (bits, huffval), (prec, name)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement writes the reference's bytes on every family
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dct", ["int", "fast", "float"])
@pytest.mark.parametrize("trellis", [[], ["-notrellis"]], ids=["trellis", "notrellis"])
def test_oracle_flat_ladder_matches_reference(built, dct, trellis):
    from oracle import oracle as O
    _need_ref("cjpeg")
    img = AC.flat_ladder()
    sw = ["-baseline", "-dct", dct] + trellis
    with tempfile.TemporaryDirectory() as d:
        for t in AC.flat_tables(Q_BASELINE_REF):
            want = _ref_pixels(img, sw + ["-qtables", _tables_file(d, t[None])])
            assert O.oracle_encode(_with_tables(_params(sw, img), t), img).jpeg == want, (dct, t[0, 0])


@pytest.mark.parametrize("dct", ["int", "float"])
def test_oracle_twelve_bit_ladder_matches_reference(built, dct):
    from oracle import oracle as O
    _need_ref("cjpeg")
    for img in (AC.flat_ladder(12), AC.gradient12()):
        sw = TWELVE + ["-dct", dct]
        with tempfile.TemporaryDirectory() as d:
            for t in AC.flat_tables(Q_WIDE, force_baseline=False):
                want = _ref_pixels(img, sw + ["-qtables", _tables_file(d, t[None])], 12)
                assert O.oracle_encode(_with_tables(_params(sw, img), t), img).jpeg == want, (dct, t[0, 0])


PIXEL_SW = {"trellis": ["-baseline"], "trellis_float": ["-baseline", "-dct", "float"], "trellis_fast": ["-baseline", "-dct", "fast"],
            "notrellis": ["-baseline", "-notrellis"], "progressive": ["-fastcrush"], "scan_search": [],
            "restart": ["-baseline", "-restart", "1"], "q95": ["-baseline", "-quality", "95"], "q100": ["-baseline", "-quality", "100"]}


@pytest.mark.parametrize("sw", list(PIXEL_SW))
def test_oracle_basis_and_screen_match_reference(built, sw):
    from oracle import oracle as O
    _need_ref("cjpeg")
    s = PIXEL_SW[sw]
    img = AC.basis_image()
    with tempfile.TemporaryDirectory() as d:
        for q in (8, 16):
            sq = s + ["-qtables", _tables_file(d, AC.flat_tables([q]))]      # scaled by -quality where given, as cjpeg does
            assert O.oracle_encode(_params(sq, img), img).jpeg == _ref_pixels(img, sq), q
    for name, im in AC.screen_images().items():
        for extra in (["-sample", "2x2"], ["-grayscale"]):
            assert O.oracle_encode(_params(s + extra, im), im).jpeg == O.ref_encode(im, s + extra), (name, extra)


@pytest.mark.parametrize("case", COEF_CASES, ids=[c[0] for c in COEF_CASES])
def test_oracle_coefficient_families_match_reference_jpegtran(built, case):
    from oracle import oracle as O
    _need_ref("jpegtran")
    _, planes, prec, tsw, scans = case
    src = _carrier(planes, prec)
    got = O.ref_read_coefs(src)["coefs"]
    assert all((g == pl).all() for g, pl in zip(got, planes))
    with tempfile.TemporaryDirectory() as d:
        sf = _scans_file(d) if scans else None
        want = O.ref_jpegtran(src, tsw + (["-scans", sf] if sf else []))
        assert _oracle_transcode(src, planes, tsw, sf) == want


def test_out_of_range_coefficient_is_refused(built):
    """One AC value of size max_coef_bits + 1: the restatement stops with JERR_BAD_DCT_COEF (jchuff.c's check)."""
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    for prec in (8, 12):
        planes = AC.out_of_range_plane(prec)
        p = mj.params_from_switches((["-precision", "12"] if prec == 12 else []) + ["-revert"], 16, 16, 1)
        with pytest.raises(RuntimeError):
            O.oracle_encode_coefs(p, planes)
        inside = [np.clip(planes[0], -(1 << (prec + 2)) + 1, (1 << (prec + 2)) - 1)]
        O.oracle_encode_coefs(p, inside)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the device writes the restatement's bytes on every family
# ---------------------------------------------------------------------------------------------------------------------
def _first_difference(enc, p, i, dbg):
    """Name the first stage where the device's debug taps differ from the restatement's."""
    for ci in range(p.num_components):
        hib, wib = dbg["hib"][ci], dbg["wib"][ci]
        for plane, key in ((1, "raw"), (2, "plain"), (0, "final")):
            try:
                dev = enc.debug_coefs(i, ci, plane)[:hib, :wib]
            except Exception:
                continue
            ref = dbg[key][ci][:hib, :wib]
            if dev.shape == ref.shape and not (dev == ref).all():
                bad = np.argwhere((dev != ref).any(-1))[0]
                return "%s coefficients of component %d differ first at block %s" % (key, ci, tuple(bad))
        for ac in (False, True):
            t = p.comp_info[ci].ac_tbl_no if ac else p.comp_info[ci].dc_tbl_no
            try:
                if enc.debug_huff(i, -1 - ci, ac, t) != dbg["trellis_ac" if ac else "trellis_dc"][ci]:
                    return "trellis-phase %s table of component %d differs" % ("AC" if ac else "DC", ci)
            except Exception:
                pass
    for s in range(dbg["nscans"]):
        for k in range(4):
            for ac in (False, True):
                want = (dbg["scan_ac"] if ac else dbg["scan_dc"])[s][k]
                try:
                    if sum(want[0]) and enc.debug_huff(i, s, ac, k) != want:
                        return "scan %d %s table %d differs" % (s, "AC" if ac else "DC", k)
                except Exception:
                    pass
    return "only the entropy-coded bytes differ"


def _check_pixels(enc, p, imgs, qt=None):
    from oracle import oracle as O
    out = enc.encode_batch(p, imgs, qtables=qt)
    for i in range(len(out)):
        pi = _with_tables(p, qt[i]) if qt is not None else p
        im = imgs[i % len(imgs)]
        want = O.oracle_encode(pi, im).jpeg
        if out[i] != want:
            dbg = O.oracle_encode(pi, im, want_debug=True).dbg
            pytest.fail("image %d: %d vs %d bytes; %s" % (i, len(out[i]), len(want), _first_difference(enc, pi, i, dbg)))


@pytest.mark.gpu
@pytest.mark.parametrize("dct", ["int", "fast", "float"])
@pytest.mark.parametrize("trellis", [[], ["-notrellis"]], ids=["trellis", "notrellis"])
def test_device_flat_ladder_every_baseline_table(encoder, dct, trellis):
    """One ladder image under 255 table sets (image stride 0): every DC and AC step 1..255 against every level."""
    img = AC.flat_ladder()
    _check_pixels(encoder, _params(["-baseline", "-dct", dct] + trellis, img), img[None], AC.flat_tables(Q_BASELINE))


WRAP_SW = [TWELVE + ["-dct", "int"], TWELVE + ["-dct", "float"]]


def test_oracle_table_value_16384_matches_reference(built):
    """A 12-bit image under a table of 16384s: the fast DCT's 16-bit scaled divisor wraps to 0 there, a table the
    integer and float DCTs quantize like any other.  (At 8 bits the reference's own reciprocal of 8 * 16384 wraps.)"""
    from oracle import oracle as O
    _need_ref("cjpeg")
    img = AC.flat_ladder(12)[:16, :16]
    with tempfile.TemporaryDirectory() as d:
        for sw in WRAP_SW:
            s = sw + ["-qtables", _tables_file(d, AC.flat_tables([16384], force_baseline=False))]
            assert O.oracle_encode(_params(s, img), img).jpeg == _ref_pixels(img, s, 12), sw


@pytest.mark.gpu
@pytest.mark.parametrize("sw", WRAP_SW, ids=["int", "float"])
def test_device_table_value_16384(encoder, sw):
    """The smallest input that stopped the encoder with SIGFPE on the host: building the fast DCT's reciprocals divided
    by the wrapped divisor whatever the DCT method."""
    img = AC.flat_ladder(12)[:16, :16]
    _check_pixels(encoder, _params(sw, img), img[None], AC.flat_tables([16384, 16], force_baseline=False))


@pytest.mark.gpu
@pytest.mark.parametrize("dct", ["int", "float"])
def test_device_twelve_bit_wide_tables(encoder, dct):
    import mozjpeg_b200 as mj
    for img in (AC.flat_ladder(12), AC.gradient12()):
        try:
            _check_pixels(encoder, _params(TWELVE + ["-dct", dct], img), img[None], AC.flat_tables(Q_WIDE, force_baseline=False))
        except mj.B200JpegError as ex:
            if ex.code != -2:
                raise
            pytest.skip("12-bit %s DCT is not on the device path" % dct)


LAYOUTS = {"gray": ["-grayscale"], "444": ["-sample", "1x1"], "422": ["-sample", "2x1"], "440": ["-sample", "1x2"],
           "420": ["-sample", "2x2"], "3x2": ["-sample", "3x2"]}


def _rgb_basis(q):
    g = np.vstack([AC.basis_image(q)] * 2)[:128, :128]
    return np.stack([g, g[:, ::-1], g[::-1]], axis=2)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("ragged", [False, True], ids=["aligned", "ragged"])
def test_device_layouts(encoder, layout, ragged):
    """Screen content and basis blocks on every tiled sampling layout and on the generic forward kernel (3x2)."""
    imgs = np.stack(list(AC.screen_images().values()) + [_rgb_basis(16)])
    if ragged:
        imgs = np.ascontiguousarray(imgs[:, :123, :117])
    _check_pixels(encoder, _params(["-baseline"] + LAYOUTS[layout], imgs[0]), imgs)


@pytest.mark.gpu
@pytest.mark.parametrize("sw", list(PIXEL_SW))
@pytest.mark.parametrize("layout", ["420", "gray"])
def test_device_switches(encoder, sw, layout):
    imgs = np.stack(list(AC.screen_images().values())[::2] + [_rgb_basis(8), _rgb_basis(16)])
    _check_pixels(encoder, _params(PIXEL_SW[sw] + LAYOUTS[layout], imgs[0]), imgs)


@pytest.mark.gpu
@pytest.mark.parametrize("sw", ["trellis", "trellis_float", "notrellis", "scan_search"])
def test_device_basis_blocks(encoder, sw):
    """Every non-zero count and the runs across 31/32 on a gray image with a coarse custom table."""
    img = AC.basis_image()
    _check_pixels(encoder, _params(PIXEL_SW[sw], img), img[None], AC.flat_tables([8, 16, 24]))


@pytest.mark.gpu
def test_device_keep_plain(built):
    """B200JPEG_KEEP_PLAIN=1 keeps the plain-quantized planes and the separate statistics pass."""
    import mozjpeg_b200 as mj
    os.environ["B200JPEG_KEEP_PLAIN"] = "1"
    try:
        e = mj.Encoder(0)
    finally:
        del os.environ["B200JPEG_KEEP_PLAIN"]
    try:
        imgs = np.stack(list(AC.screen_images().values()) + [_rgb_basis(16)])
        for layout in ("420", "gray", "3x2"):
            _check_pixels(e, _params(["-baseline"] + LAYOUTS[layout], imgs[0]), imgs)
        img = AC.basis_image()
        _check_pixels(e, _params(["-baseline"], img), img[None], AC.flat_tables([8, 16]))
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [1, 2])
def test_device_chunked_batches(built, chunk):
    import mozjpeg_b200 as mj
    imgs = np.stack(list(AC.screen_images().values())[:5])
    e = mj.Encoder(0)
    try:
        e.set_chunk_images(chunk)
        for sw in (["-baseline", "-sample", "2x2", "-restart", "1"], ["-fastcrush", "-sample", "2x2"]):
            _check_pixels(e, _params(sw, imgs[0]), imgs)
        img = AC.flat_ladder()
        _check_pixels(e, _params(["-baseline"], img), img[None], AC.flat_tables([1, 16, 17, 255, 64]))
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", COEF_CASES, ids=[c[0] for c in COEF_CASES])
def test_device_coefficient_families(encoder, case):
    _, planes, prec, tsw, scans = case
    src = _carrier(planes, prec)
    with tempfile.TemporaryDirectory() as d:
        sf = _scans_file(d) if scans else None
        p, _ = _transcode_params(src, tsw, sf)
        from oracle import oracle as O
        want = O.oracle_encode_coefs(p, planes)
        got = encoder.encode_batch_coefs(p, [a[None] for a in planes])[0]
    assert got == want, (len(got), len(want))


@pytest.mark.gpu
def test_device_out_of_range_coefficient(encoder):
    """The device reports JERR_BAD_DCT_COEF like the reference, and the same encoder then encodes the next batch."""
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    from oracle import oracle as O
    for prec in (8, 12):
        planes = AC.out_of_range_plane(prec)
        inside = [np.clip(planes[0], -(1 << (prec + 2)) + 1, (1 << (prec + 2)) - 1)]
        src = _carrier(inside, prec)
        for tsw in (["-revert"], ["-revert", "-optimize"], ["-progressive"]):
            p, _ = _transcode_params(src, tsw)
            with pytest.raises(mj.B200JpegError) as ex:
                encoder.encode_batch_coefs(p, [a[None] for a in planes])
            assert ex.value.code == A.ERR_BAD_DCT_COEF
            assert encoder.encode_batch_coefs(p, [a[None] for a in inside])[0] == O.oracle_encode_coefs(p, inside)
