"""Device entropy decode of sequential Huffman JPEG files (b200jpeg_decode_coefs_batch / b200jpeg_transcode_batch) and
the source-header parser behind it (b200jpeg_parse_source).  Sources come from tests/decode_cases.py; the md5s of the
reference's jpeg_read_coefficients planes are in tests/golden/decode_golden.json (tools/make_golden.py --decode)."""
import hashlib
import json
import os
import struct

import numpy as np
import pytest

import decode_cases as D
from common import GOLD

GD = {c["id"]: c for c in json.load(open(os.path.join(GOLD, "decode_golden.json")))["cases"]}
TR = json.load(open(os.path.join(GOLD, "transcode_golden.json")))["cases"]
_cache = {}


def _src(case):
    if case[0] not in _cache:
        _cache.clear()
        _cache[case[0]] = D.source(case)
    return _cache[case[0]]


def _markers(jpeg: bytes):
    """(marker, offset) of every marker segment before the first SOS's data, for building edited files"""
    out, pos = [], 2
    while pos < len(jpeg):
        m = jpeg[pos + 1]
        ln = struct.unpack(">H", jpeg[pos + 2:pos + 4])[0]
        out.append((m, pos))
        if m == 0xDA:
            break
        pos += 2 + ln
    return out


def _sos_data(jpeg: bytes):
    from mozjpeg_b200 import jpegtran as T
    s = T.parse_source(jpeg).scans[0]
    return s.data_offset, s.data_size


def _seg(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


ALL_IDS = [c[0] for c in D.CASES] + D.EXTRA_IDS


def _src_bytes(name):
    byid = {c[0]: c for c in D.CASES}
    return _src(byid[name])[0] if name in byid else D.extra_source(name)


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("case", D.CASES, ids=[c[0] for c in D.CASES])
def test_sources_match_recorded_files_and_reference_planes(built, case):
    src, planes = _src(case)
    assert hashlib.md5(src).hexdigest() == GD[case[0]]["src_md5"]
    assert D.md5_planes(planes) == GD[case[0]]["coef_md5"]


@pytest.mark.parametrize("name", D.EXTRA_IDS)
def test_constructed_sources_match_recorded_files(built, name):
    from oracle import oracle as O
    src = D.extra_source(name)
    assert hashlib.md5(src).hexdigest() == GD[name]["src_md5"]
    if O.ref_available():
        assert D.md5_planes(O.ref_read_coefs(src)["coefs"]) == GD[name]["coef_md5"]


def test_parser_installs_standard_tables_where_the_file_has_none(built):
    """std_huff_tables (jdhuff.c:819-823): a sequential file without DHT reads with the standard tables in slots 0 and
    1; slots 2 and 3 stay undefined, and a progressive reader installs nothing (jdphuff.c)."""
    import ctypes
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T, _abi as A
    from oracle import oracle as O
    src = D.extra_source("no_dht")
    r = T.parse_source(src)
    assert r.num_huff == 4 and sorted(r.huff_is_dc[:4]) == [0, 0, 1, 1]
    p = mj.Params(); A.load().b200jpeg_std_huff_tables(ctypes.byref(p))
    sc = r.scans[0]
    for i in range(3):
        t = sc.dc_tbl_no[i]
        assert bytes(r.huff[sc.dc_huff[i]].bits) == bytes(p.dc_huff_tbl[t].bits) and bytes(r.huff[sc.ac_huff[i]].huffval) == bytes(p.ac_huff_tbl[t].huffval)
    assert T.parse_header(src).comps == T.parse_header(_src(D.CASES[0])[0]).comps
    lib = A.load()
    bad = bytearray(src); k = _markers(src)[-1][1]; bad[k + 6] = 0x22                             # component 1 names slot 2
    assert lib.b200jpeg_parse_source(bytes(bad), len(bad), ctypes.byref(A.SourceInfo())) == A.ERR_BAD_SOURCE
    prog = D._strip_dht(O.oracle_encode(mj.params_from_switches(["-progressive", "-revert"], 64, 48, 3), D.pixels(3, 64, 48)).jpeg)
    assert lib.b200jpeg_parse_source(prog, len(prog), ctypes.byref(A.SourceInfo())) == A.ERR_BAD_SOURCE


def test_fill_bytes_inside_entropy_coded_data_end_it(built):
    """FF FF 00 is not a stuffed 0xFF: fill bytes may only precede a marker, and the reference's decoder hits a marker
    there; the data ends, and what follows is no marker, so the file is refused"""
    import ctypes
    from mozjpeg_b200 import jpegtran as T, _abi as A
    src = D.extra_source("carrier_ff")
    sc = T.parse_source(src).scans[0]
    k = src.index(b"\xff\x00", sc.data_offset)
    bad = src[:k] + b"\xff" + src[k:]
    assert A.load().b200jpeg_parse_source(bad, len(bad), ctypes.byref(A.SourceInfo())) == A.ERR_BAD_SOURCE
    assert b"0x00" in A.load().b200jpeg_last_error()


@pytest.mark.parametrize("case", D.CASES[:12] + D.CASES[13:15], ids=[c[0] for c in D.CASES[:12] + D.CASES[13:15]])
def test_parser_fields(built, case):
    """b200jpeg_parse_source against the parameter block the file was written from, and parse_header built on it."""
    from mozjpeg_b200 import jpegtran as T, _abi as A
    from oracle import oracle as O
    src, _ = _src(case)
    p = D.params(case)
    r = T.parse_source(src)
    assert (r.sof, r.image_width, r.image_height, r.data_precision, r.num_components) == (0xC0, p.image_width, p.image_height, 8, p.num_components)
    for ci in range(p.num_components):
        c = p.comp_info[ci]
        assert (r.component_id[ci], r.h_samp_factor[ci], r.v_samp_factor[ci], r.quant_tbl_no[ci]) == (c.component_id, c.h_samp_factor, c.v_samp_factor, c.quant_tbl_no)
        assert list(r.comp_quant[ci]) == list(p.quant_tbl[c.quant_tbl_no])
    assert r.num_scans == (p.num_scans or 1)
    ri = p.restart_interval or (p.restart_in_rows * -(-p.image_width // (8 * max(c.h_samp_factor for c in p.comp_info[:p.num_components]))))
    assert all(r.scans[k].restart_interval == ri for k in range(r.num_scans))
    assert r.scans[r.num_scans - 1].data_offset + r.scans[r.num_scans - 1].data_size == len(src) - 2       # EOI follows
    h = T.parse_header(src)
    assert h.comps == [(r.component_id[i], r.h_samp_factor[i], r.v_samp_factor[i], r.quant_tbl_no[i]) for i in range(r.num_components)]
    assert h.jpeg_color_space == (A.CS_RGB if "-rgb" in case[4] else A.CS_GRAYSCALE if "-grayscale" in case[4] else A.CS_YCbCr)
    if O.ref_available():
        ref = O.ref_read_coefs(src)
        assert [a.shape[:2] for a in ref["coefs"]] == [(-(-p.image_height * c.v_samp_factor // (8 * max(x.v_samp_factor for x in p.comp_info[:p.num_components]))),
                                                        -(-p.image_width * c.h_samp_factor // (8 * max(x.h_samp_factor for x in p.comp_info[:p.num_components]))))
                                                       for c in p.comp_info[:p.num_components]]


def test_parser_edge_headers(built):
    """16-bit DQT, SOF2, DHT between scans, fill bytes before markers and a DNL marker after the scan parse like the
    reference reads them."""
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    src, _ = _src(D.CASES[13])                                  # three sequential scans, tables before the first
    r = T.parse_source(src)
    assert r.num_scans == 3 and [r.scans[k].component_index[0] for k in range(3)] == [0, 1, 2]
    # fill bytes before every marker after the first scan, and a DNL marker behind the last scan
    end0 = r.scans[0].data_offset + r.scans[0].data_size
    last = r.scans[2].data_offset + r.scans[2].data_size
    dnl = _seg(0xDC, struct.pack(">H", r.image_height))
    edited = src[:end0] + b"\xff\xff\xff" + src[end0:last] + dnl + b"\xff\xff" + src[last:]
    e = T.parse_source(edited)
    assert e.num_scans == 3 and e.scans[0].data_size == r.scans[0].data_size and e.scans[2].data_size == r.scans[2].data_size
    # a DHT between scans: the second scan uses the definition in force at its SOS
    sos1 = r.scans[1].data_offset - (6 + 2 * 1) - 2
    bits = bytes([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0])
    dht = _seg(0xC4, bytes([0x01]) + bits + bytes(range(12)))
    e = T.parse_source(src[:sos1] + dht + src[sos1:])
    assert e.scans[1].dc_huff[0] == e.num_huff - 1 and e.scans[0].dc_huff[0] != e.num_huff - 1
    # 16-bit DQT
    info = T.parse_header(src)
    q16 = bytes([0x10 | 2]) + b"".join(struct.pack(">H", 300 + k) for k in range(64))
    e = T.parse_source(src[:2] + _seg(0xDB, q16) + src[2:])
    assert e.quant_tbl_present[2] and e.quant_tbl[2][0] == 300 and e.quant_tbl[2][63] == 363
    assert T.parse_header(src).quant == info.quant
    # SOF2: parsed, every scan recorded
    prog = O.oracle_encode(__import__("mozjpeg_b200").params_from_switches(["-progressive", "-revert"], 64, 48, 3), D.pixels(3, 64, 48)).jpeg
    e = T.parse_source(prog)
    assert e.sof == 0xC2 and e.num_scans > 3


def test_parser_refusals(built):
    from mozjpeg_b200 import jpegtran as T, _abi as A
    lib = A.load()
    src, _ = _src(D.CASES[0])
    marks = dict((m, o) for m, o in _markers(src))
    sof = marks[0xC0]

    def code(b):
        return lib.b200jpeg_parse_source(b, len(b), __import__("ctypes").byref(A.SourceInfo()))

    assert code(src) == 0
    for m, want in ((0xC3, A.ERR_UNSUPPORTED), (0xC9, A.ERR_UNSUPPORTED)):
        assert code(src[:sof + 1] + bytes([m]) + src[sof + 2:]) == want
    assert code(src[:sof + 5] + b"\x00\x00" + src[sof + 7:]) == A.ERR_BAD_SOURCE                  # height 0
    assert code(src[:sof + 9]) == A.ERR_PARAM                                                    # the file ends inside the SOF
    sos = marks[0xDA]
    bad_sel = bytearray(src); bad_sel[sos + 6] = 0x33                                             # component 1 names DC/AC table 3
    assert code(bytes(bad_sel)) == A.ERR_BAD_SOURCE
    with pytest.raises(ValueError):
        T.parse_header(b"\x00\x01")


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", ALL_IDS)
def test_read_coefficients_matches_reference(encoder, name):
    got = encoder.read_coefficients([_src_bytes(name)])
    assert D.md5_planes([a[0] for a in got]) == GD[name]["coef_md5"]


@pytest.mark.gpu
def test_transcode_of_a_file_without_dht(encoder):
    from mozjpeg_b200 import jpegtran as T
    src = _src(D.CASES[0])[0]
    for tsw in ([], ["-revert", "-optimize"]):
        assert T.transcode(encoder, [D.extra_source("no_dht")], None, tsw) == T.transcode(encoder, [src], None, tsw)


def _seq_sources():
    """the recorded cases whose source is sequential: mozjpeg's cjpeg writes progressive files unless -revert or
    -baseline turns that off"""
    for c in TR:
        if ("-revert" in c["enc"] or "-baseline" in c["enc"]) and "-progressive" not in c["enc"]:
            yield c


@pytest.mark.gpu
@pytest.mark.parametrize("c", list(_seq_sources()), ids=lambda c: "%dx%d:%s:%s" % (c["width"], c["height"], "_".join(s.lstrip("-") for s in c["enc"]), "_".join(s.lstrip("-") for s in c["tran"]) or "default"))
def test_transcode_from_file_bytes_matches_recorded_jpegtran(encoder, c):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    im = O.synth_image(c["seed"], c["width"], c["height"])
    src = O.oracle_encode(mj.params_from_switches(c["enc"], c["width"], c["height"], 3), im).jpeg
    assert hashlib.md5(src).hexdigest() == c["src_md5"]
    out = T.transcode(encoder, [src], None, c["tran"])[0]
    assert len(out) == c["size"] and hashlib.md5(out).hexdigest() == c["md5"]


def _mixed_batch():
    """same geometry; different Huffman tables, quantization tables, restart intervals and scan layouts"""
    cases = [("a", 200, 136, 31, ["-revert"], None), ("b", 200, 136, 32, ["-revert", "-optimize", "-restart", "2B"], None),
             ("c", 200, 136, 33, ["-revert", "-quality", "40"], "multi"), ("d", 200, 136, 34, ["-revert", "-quality", "70", "-restart", "1"], None),
             ("e", 200, 136, 35, ["-revert", "-optimize", "-quality", "60"], "multi")]
    return [D.source(c) for c in cases]


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 2])
def test_mixed_batch_equals_single_images(encoder, chunk):
    from mozjpeg_b200 import jpegtran as T
    srcs = [s for s, _ in _mixed_batch()]
    for tsw in ([], ["-optimize"], ["-progressive"]):
        singles = [T.transcode(encoder, [s], None, tsw)[0] for s in srcs]
        encoder.set_chunk_images(chunk)
        try:
            batch = T.transcode(encoder, srcs, None, tsw)
        finally:
            encoder.set_chunk_images(0)
        assert batch == singles, tsw
    got = encoder.read_coefficients(srcs)
    for i, (_, planes) in enumerate(_mixed_batch()):
        for ci, a in enumerate(planes):
            assert np.array_equal(got[ci][i], a), (i, ci)


@pytest.mark.gpu
def test_round_trip_of_device_encoded_files(encoder):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    w, h = 328, 200
    for sw in (["-baseline", "-quality", "80"], ["-revert", "-quality", "90", "-restart", "1", "-sample", "2x1"], ["-baseline", "-quality", "60", "-grayscale"]):
        penc = mj.params_from_switches(sw, w, h, 3)
        imgs = np.stack([O.synth_image(40 + i, w, h) for i in range(3)])
        files = encoder.encode_batch(penc, imgs if penc.input_components == 3 else imgs[..., 0])
        planes = encoder.read_coefficients(files)
        q = penc.copy(); q.trellis_quant = 0
        assert encoder.encode_batch_coefs(q, planes) == files, sw


def _expect_bad(encoder, files, image):
    from mozjpeg_b200 import _abi as A
    with pytest.raises(A.B200JpegError) as ei:
        encoder.read_coefficients(files)
    assert ei.value.code == A.ERR_BAD_SOURCE and f"image {image}" in str(ei.value)


@pytest.mark.gpu
def test_malformed_files_are_refused_and_the_encoder_recovers(encoder):
    good, planes = _src(D.CASES[0])
    off, size = _sos_data(good)
    truncated = good[:off + size // 2]
    invalid = good[:off + size // 2] + b"\xff\x00" * 8 + good[off + size // 2 + 16:]
    rst_src, _ = D.source(D.CASES[8])
    k = rst_src.index(b"\xff\xd1", _sos_data(rst_src)[0])
    wrong_rst = rst_src[:k + 1] + b"\xd5" + rst_src[k + 2:]
    garbage = good[:off + size] + bytes(range(1, 200)) + good[off + size:]
    _expect_bad(encoder, [good, truncated], 1)
    _expect_bad(encoder, [invalid, good], 0)
    _expect_bad(encoder, [rst_src, wrong_rst], 1)
    k = good.index(b"\xff\x00", off)
    _expect_bad(encoder, [good[:k] + b"\xff" + good[k:]], 0)           # FF FF 00 inside the data: a marker hit
    got = encoder.read_coefficients([garbage])                  # bytes after the last MCU are ignored, like the reference
    assert all(np.array_equal(g[0], a) for g, a in zip(got, planes))
    got = encoder.read_coefficients([good, good])
    assert all(np.array_equal(g[1], a) for g, a in zip(got, planes))
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    p = mj.params_from_switches(["-quality", "75"], 64, 48, 3)
    im = O.synth_image(1, 64, 48)
    assert encoder.encode_batch(p, im[None])[0] == O.oracle_encode(p, im).jpeg


@pytest.mark.gpu
def test_progressive_source_points_to_the_planes_form(encoder):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T, _abi as A
    from oracle import oracle as O
    prog = O.oracle_encode(mj.params_from_switches(["-progressive", "-revert"], 64, 48, 3), D.pixels(3, 64, 48)).jpeg
    with pytest.raises(A.B200JpegError) as ei:
        encoder.read_coefficients([prog])
    assert ei.value.code == A.ERR_UNSUPPORTED
    with pytest.raises(ValueError, match="coef_planes"):
        T.transcode(encoder, [prog], None, [])


@pytest.mark.gpu
def test_jpegtran_command_line(encoder, tmp_path):
    from mozjpeg_b200 import jpegtran as T
    src, _ = _src(D.CASES[0])
    (tmp_path / "in.jpg").write_bytes(src)
    assert T.main(["-optimize", "-outfile", str(tmp_path / "o.jpg"), str(tmp_path / "in.jpg")]) == 0
    assert (tmp_path / "o.jpg").read_bytes() == T.transcode(encoder, [src], None, ["-optimize"])[0]
    st = encoder.stage_times()
    assert all(k in st for k in ("dec_h2d", "dec_sync", "dec_fix", "dec_scan", "dec_write", "dec_dc"))
