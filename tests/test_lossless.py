"""Lossless JPEG (SOF3) at 8, 12 and 16 bits: parameter logic against the reference on the CPU, and the device path byte
for byte against the unmodified reference library (oracle/_ref through tests/refll.c, built by __graft_entry__.build())."""
import ctypes as C
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import mozjpeg_b200 as mj
from mozjpeg_b200 import _abi as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFLL = os.path.join(ROOT, "build", "librefll.so")
# the reference's bytes for every case below (tools/make_golden.py --lossless, which also checks them against the
# reference's own cjpeg binary wherever it can read the input)
GOLDEN = {c["id"]: c["md5"] for c in json.load(open(os.path.join(ROOT, "tests", "golden", "lossless_golden.json")))["cases"]}
lib = A.load()

CS_EXT = {"EXT_RGB": (6, 3), "EXT_RGBX": (7, 4), "EXT_BGR": (8, 3), "EXT_BGRX": (9, 4), "EXT_XBGR": (10, 4),
          "EXT_XRGB": (11, 4), "EXT_RGBA": (12, 4), "EXT_BGRA": (13, 4), "EXT_ABGR": (14, 4), "EXT_ARGB": (15, 4)}

_ref = None


def refll():
    global _ref
    if _ref is None:
        if not os.path.exists(REFLL):
            pytest.skip("the reference build (oracle/_ref) is not present")
        _ref = C.CDLL(REFLL)
        _ref.refll_encode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_char_p),
                                      C.c_int, C.POINTER(C.c_int), C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_ulong), C.c_char_p, C.c_int]
        _ref.refll_free.argtypes = [C.c_void_p]
    return _ref


def ref_encode(pix, switches, in_cs, script=None):
    """The reference's bytes, or the reference's error message as a RuntimeError."""
    h, w, nc = pix.shape
    argv = (C.c_char_p * max(1, len(switches)))(*[s.encode() for s in switches])
    flat = [v for (comps, ss, al) in (script or []) for v in ([len(comps)] + list(comps) + [0] * (4 - len(comps)) + [ss, 0, 0, al])]
    sc = (C.c_int * max(1, len(flat)))(*flat)
    out = C.POINTER(C.c_uint8)(); n = C.c_ulong(0); err = C.create_string_buffer(256)
    rc = refll().refll_encode(pix.ctypes.data, pix.strides[0] // pix.itemsize, w, h, in_cs, nc, len(switches), argv,
                              len(script or []), sc, C.byref(out), C.byref(n), err, 256)
    if rc:
        raise RuntimeError(err.value.decode())
    data = C.string_at(out, n.value)
    refll().refll_free(out)
    return data


def params(switches, w, h, nc, in_cs, script=None):
    p = mj.params_from_switches(switches, w, h, nc, in_color_space=in_cs)
    if script:
        p.num_scans = len(script)
        for i, (comps, ss, al) in enumerate(script):
            e = p.scan_info[i]
            e.comps_in_scan = len(comps)
            for k in range(4):
                e.component_index[k] = comps[k] if k < len(comps) else 0
            e.Ss, e.Se, e.Ah, e.Al = ss, 0, 0, al
        p.optimize_scans = 0
    return p


def image(seed, h, w, nc, prec, kind="smooth"):
    rng = np.random.default_rng(seed)
    top = (1 << prec) - 1
    if kind == "alternating":                                     # 0 / max: every difference is +-max (category 16 at 16 bits)
        a = ((np.indices((h, w)).sum(axis=0) % 2) * top)[..., None].repeat(nc, axis=2)
    elif kind == "wide12":                                        # 12-bit rows holding values above 4095 (J12SAMPLE is signed)
        a = rng.integers(0, 65536, size=(h, w, nc))
    else:
        yy, xx = np.mgrid[0:h, 0:w]
        base = (xx * 7 + yy * 3)[..., None] * (top // 255 + 1) + np.arange(nc) * 17
        a = (base + rng.integers(0, max(2, top // 64), size=(h, w, nc))) % (top + 1)
    return np.ascontiguousarray(a, dtype=np.uint8 if prec == 8 else np.uint16)


# (switches, in_color_space, components, precision, (h, w), kind, script)
CASES = []
for prec in (8, 12, 16):
    for psv in range(1, 8):
        for pt in sorted({0, 1, prec - 1}):
            CASES.append((["-revert", "-precision", str(prec), "-lossless", f"{psv},{pt}"], A.CS_GRAYSCALE, 1, prec, (19, 23), "smooth", None))
for name, (cs, nc) in CS_EXT.items():
    CASES.append((["-revert", "-lossless", "4"], cs, nc, 8, (17, 29), "smooth", None))
CASES += [
    (["-revert", "-lossless", "1"], A.CS_RGB, 3, 8, (37, 53), "smooth", None),
    (["-revert", "-precision", "12", "-lossless", "6,2"], A.CS_RGB, 3, 12, (21, 30), "smooth", None),
    (["-revert", "-precision", "16", "-lossless", "7,1"], A.CS_RGB, 3, 16, (21, 30), "smooth", None),
    (["-revert", "-lossless", "2"], A.CS_CMYK, 4, 8, (13, 22), "smooth", None),
    (["-revert", "-precision", "16", "-lossless", "3"], A.CS_YCCK, 4, 16, (13, 22), "smooth", None),
    (["-revert", "-lossless", "5,1"], A.CS_YCbCr, 3, 8, (13, 22), "smooth", None),
    (["-revert", "-precision", "12", "-lossless", "1"], A.CS_UNKNOWN, 2, 12, (13, 22), "smooth", None),
    # the trap rows: switches the start-time overrides undo, and the default profile's multi-table markers
    (["-revert", "-lossless", "1", "-grayscale"], A.CS_RGB, 3, 8, (16, 16), "smooth", None),
    (["-revert", "-lossless", "1", "-rgb"], A.CS_RGB, 3, 8, (16, 16), "smooth", None),
    (["-revert", "-lossless", "1", "-sample", "2x2"], A.CS_RGB, 3, 8, (16, 16), "smooth", None),
    (["-revert", "-lossless", "1", "-smooth", "30"], A.CS_RGB, 3, 8, (16, 16), "smooth", None),
    (["-baseline", "-notrellis", "-lossless", "2"], A.CS_RGB, 3, 8, (16, 16), "smooth", None),
    (["-baseline", "-notrellis", "-lossless", "2"], A.CS_YCbCr, 3, 8, (16, 16), "smooth", None),
    (["-revert", "-precision", "16", "-lossless", "5,3"], A.CS_GRAYSCALE, 1, 16, (31, 17), "smooth", None),
    (["-revert", "-progressive", "-lossless", "1"], A.CS_RGB, 3, 8, (16, 16), "smooth", None),      # progressive script wins
    # restarts: 1, 2 and 7 rows, in rows and in MCUs
    (["-revert", "-lossless", "4", "-restart", "1"], A.CS_RGB, 3, 8, (23, 53), "smooth", None),
    (["-revert", "-lossless", "4", "-restart", "2"], A.CS_GRAYSCALE, 1, 8, (23, 53), "smooth", None),
    (["-revert", "-precision", "16", "-lossless", "6", "-restart", "7"], A.CS_GRAYSCALE, 1, 16, (23, 53), "smooth", None),
    (["-revert", "-lossless", "4", "-restart", "53B"], A.CS_RGB, 3, 8, (23, 53), "smooth", None),
    (["-revert", "-lossless", "7", "-restart", "106B"], A.CS_RGB, 3, 8, (23, 53), "smooth", None),
    (["-revert", "-precision", "12", "-lossless", "2", "-restart", "371B"], A.CS_GRAYSCALE, 1, 12, (23, 53), "smooth", None),
    # hand-made scripts: one component per scan, different predictors and point transforms, two scans
    (["-revert"], A.CS_RGB, 3, 8, (19, 27), "smooth", [((0,), 1, 0), ((1,), 3, 1), ((2,), 7, 2)]),
    (["-revert", "-precision", "16"], A.CS_RGB, 3, 16, (19, 27), "smooth", [((0, 2), 6, 0), ((1,), 5, 4)]),
    (["-revert", "-restart", "2"], A.CS_CMYK, 4, 8, (19, 27), "smooth", [((1, 3), 4, 0), ((0, 2), 2, 1)]),
    # ragged shapes
    (["-revert", "-lossless", "4"], A.CS_GRAYSCALE, 1, 8, (1, 1), "smooth", None),
    (["-revert", "-lossless", "4"], A.CS_RGB, 3, 8, (1, 40), "smooth", None),
    (["-revert", "-lossless", "4"], A.CS_RGB, 3, 8, (40, 1), "smooth", None),
    (["-revert", "-precision", "16", "-lossless", "6"], A.CS_GRAYSCALE, 1, 16, (3, 65500), "smooth", None),
    (["-revert", "-lossless", "5"], A.CS_GRAYSCALE, 1, 8, (65500, 3), "smooth", None),
    # extreme content
    (["-revert", "-precision", "16", "-lossless", "1"], A.CS_GRAYSCALE, 1, 16, (20, 21), "alternating", None),
    (["-revert", "-precision", "16", "-lossless", "4"], A.CS_RGB, 3, 16, (20, 21), "alternating", None),
    (["-revert", "-lossless", "7"], A.CS_GRAYSCALE, 1, 8, (20, 21), "alternating", None),
    (["-revert", "-precision", "12", "-lossless", "4"], A.CS_GRAYSCALE, 1, 12, (20, 21), "wide12", None),
    (["-revert", "-precision", "12", "-lossless", "6,3"], A.CS_RGB, 3, 12, (20, 21), "wide12", None),
    (["-revert", "-precision", "16", "-lossless", "2"], A.CS_RGB, 3, 16, (20, 21), "wide12", None),
]


def _id(c):
    sw, cs, nc, prec, (h, w), kind, script = c
    return f"{' '.join(sw)}|cs{cs}x{nc}|p{prec}|{h}x{w}|{kind}" + ("|script" if script else "")


# ---------------------------------------------------------------- CPU: parameter logic
def test_enable_lossless_script_and_ranges():
    p = mj.params_from_switches(["-revert"], 32, 16, 3)
    assert lib.b200jpeg_enable_lossless(C.byref(p), 0, 0) == A.ERR_PARAM
    assert lib.b200jpeg_enable_lossless(C.byref(p), 8, 0) == A.ERR_PARAM
    assert lib.b200jpeg_enable_lossless(C.byref(p), 1, 8) == A.ERR_PARAM
    assert lib.b200jpeg_enable_lossless(C.byref(p), 3, 2) == 0
    s = p.scan_info[0]
    assert p.num_scans == 1 and s.comps_in_scan == 3 and list(s.component_index)[:3] == [0, 1, 2] and (s.Ss, s.Se, s.Ah, s.Al) == (3, 0, 0, 2)
    assert lib.b200jpeg_validate(C.byref(p)) == 0
    assert lib.b200jpeg_total_passes(C.byref(p)) == 2                     # optimize_coding forced: 2 passes per scan
    assert p.scan_info[1].comps_in_scan == -1                                 # marks the stand-in for scan_info == NULL
    assert lib.b200jpeg_enable_lossless(C.byref(p), 6, 1) == 0                # a second call overwrites, as in the reference
    assert p.num_scans == 1 and (p.scan_info[0].Ss, p.scan_info[0].Al) == (6, 1)
    # beside the scan search's script the reference keeps lossless mode on next to progressive mode
    q = mj.params_from_switches([], 32, 16, 3)
    assert q.num_scans > 0 and lib.b200jpeg_enable_lossless(C.byref(q), 1, 0) == A.ERR_PARAM              # trellis on
    q.trellis_quant = 0
    assert lib.b200jpeg_enable_lossless(C.byref(q), 1, 0) == A.ERR_UNSUPPORTED                            # SOF2 over lossless data
    # over any other script validate_script decides: a progressive script turns lossless off, the call changes nothing
    r = mj.params_from_switches(["-revert", "-progressive"], 32, 16, 3)
    before = bytes(r)
    assert lib.b200jpeg_enable_lossless(C.byref(r), 1, 0) == 0 and bytes(r) == before


def test_hand_made_one_scan_script_is_kept():
    # a hand-installed script of component 0 is not the stand-in for scan_info == NULL: the colour-space override does
    # not widen it (the reference codes the one scan it was given)
    p = params(["-revert", "-grayscale"], 32, 16, 3, A.CS_RGB, [((0,), 1, 0)])
    assert p.num_components == 1 and lib.b200jpeg_validate(C.byref(p)) == 0
    q = mj.params_from_switches(["-revert", "-grayscale", "-lossless", "1"], 32, 16, 3)
    assert q.scan_info[1].comps_in_scan == -1 and lib.b200jpeg_validate(C.byref(q)) == 0


def test_default_colorspace_and_simple_progression_follow_lossless():
    p = mj.params_from_switches(["-revert", "-lossless", "1"], 32, 16, 3)
    assert p.jpeg_color_space == A.CS_YCbCr                                   # cjpeg ran default_colorspace before the lossless switch took effect
    assert lib.b200jpeg_default_colorspace(C.byref(p)) == 0 and p.jpeg_color_space == A.CS_RGB     # jcparam.c:544-549
    assert lib.b200jpeg_simple_progression(C.byref(p)) == 0                  # jcparam.c:875-880: lossless off again
    assert p.jpeg_color_space == A.CS_YCbCr and p.num_scans > 1 and p.scan_info[0].Se == 0 and p.scan_info[0].Ss == 0


def test_validate_error_classes():
    def rc(p):
        return lib.b200jpeg_validate(C.byref(p))
    assert rc(mj.params_from_switches(["-revert", "-precision", "16"], 32, 16, 3)) == A.ERR_PARAM           # 16-bit lossy (jcinit.c:95-96)
    p = mj.params_from_switches(["-revert", "-lossless", "1"], 32, 16, 3)
    p.trellis_quant = 1
    assert rc(p) == A.ERR_PARAM                                                                            # "Bogus buffer control mode"
    assert rc(mj.params_from_switches(["-baseline", "-lossless", "2"], 32, 16, 3)) == A.ERR_PARAM          # default profile: trellis on
    with pytest.raises(mj.B200JpegError) as ei:                                                           # default profile, scan search script
        mj.params_from_switches(["-lossless", "1"], 32, 16, 3)
    assert ei.value.code == A.ERR_PARAM
    with pytest.raises(mj.B200JpegError) as ei:
        mj.params_from_switches(["-notrellis", "-lossless", "1"], 32, 16, 3)
    assert ei.value.code == A.ERR_UNSUPPORTED
    assert rc(mj.params_from_switches(["-revert", "-lossless", "4", "-restart", "40B"], 53, 16, 3)) == A.ERR_PARAM   # JERR_BAD_RESTART
    assert rc(mj.params_from_switches(["-revert", "-lossless", "4", "-restart", "106B"], 53, 16, 3)) == 0
    p = mj.params_from_switches(["-revert", "-lossless", "1"], 32, 16, 3)
    p.input_components = 4
    assert rc(p) == A.ERR_PARAM                                                                            # Bogus input colorspace
    p = params(["-revert"], 32, 16, 3, A.CS_RGB, [((0,), 1, 0), ((1,), 1, 0)])
    assert rc(p) == A.ERR_PARAM                                                                            # component 2 never sent
    p = params(["-revert"], 32, 16, 3, A.CS_RGB, [((0, 1, 2), 1, 8)])
    assert rc(p) == A.ERR_PARAM                                                                            # Al >= precision
    p = params(["-revert"], 32, 16, 3, A.CS_RGB, [((0, 1), 1, 0), ((1, 2), 1, 0)])
    assert rc(p) == A.ERR_PARAM                                                                            # component sent twice
    assert lib.b200jpeg_total_passes(C.byref(params(["-revert"], 32, 16, 3, A.CS_RGB, [((0,), 1, 0), ((1,), 2, 0), ((2,), 3, 0)]))) == 6


@pytest.mark.parametrize("switches,w", [(["-revert", "-lossless", "4", "-restart", "40B"], 53), (["-baseline", "-lossless", "2"], 16),
                                        (["-revert", "-precision", "16"], 16), (["-revert", "-lossless", "1"], 16)])
def test_validate_agrees_with_reference(switches, w):
    pix = image(1, 8, w, 3, 16 if "16" in switches else 8)
    try:
        ref_encode(pix, switches, A.CS_RGB)
        ref_ok = True
    except RuntimeError:
        ref_ok = False
    p = mj.params_from_switches(switches, w, 8, 3)
    assert (lib.b200jpeg_validate(C.byref(p)) == 0) == ref_ok


def test_cjpeg_mirror_trap_rows():
    base = mj.params_from_switches(["-revert", "-lossless", "1"], 16, 16, 3)
    for extra in (["-grayscale"], ["-rgb"], ["-sample", "2x2"], ["-smooth", "30"]):
        p = mj.params_from_switches(["-revert", "-lossless", "1"] + extra, 16, 16, 3)
        assert lib.b200jpeg_validate(C.byref(p)) == 0
        s = p.scan_info[0]
        assert p.num_scans == 1 and (s.Ss, s.Se, s.Al) == (1, 0, 0)
    q = mj.params_from_switches(["-revert", "-precision", "16", "-lossless", "5,3"], 16, 16, 1)
    assert q.data_precision == 16 and (q.scan_info[0].Ss, q.scan_info[0].Al) == (5, 3) and lib.b200jpeg_validate(C.byref(q)) == 0
    assert base.optimize_scans == 0


def test_read_pnm_16bit_and_maxval_refusal():
    a = np.array([[1, 65535, 300]], dtype=np.uint16)
    f = b"P5\n3 1\n65535\n" + a.astype(">u2").tobytes()
    w, h, nc, maxv, s = mj.read_pnm(f)
    assert (w, h, nc, maxv) == (3, 1, 1, 65535) and s.dtype == np.uint16 and np.array_equal(s.ravel(), a.ravel())
    assert mj.pnm_samples(maxv, s, 16) is s
    # rdppm.c would rescale these samples: refused rather than coded with values the reference does not see
    for prec in (8, 12):
        with pytest.raises(ValueError):
            mj.pnm_samples(maxv, s, prec)
    with pytest.raises(ValueError):
        mj.cjpeg(["-revert", "-lossless", "1"], f)
    with pytest.raises(ValueError):
        mj.read_ppm(f)                                                          # the 8-bit reader stays 8-bit


def test_reference_driver_matches_golden():
    for c in CASES:
        sw, cs, nc, prec, (h, w), kind, script = c
        pix = image(zlib.crc32(_id(c).encode()), h, w, nc, prec, kind)
        assert hashlib.md5(ref_encode(pix, sw, cs, script)).hexdigest() == GOLDEN[_id(c)], _id(c)


# ---------------------------------------------------------------- GPU: byte-identical to the reference
@pytest.fixture(scope="module")
def enc():
    e = mj.Encoder(0)
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_id)
def test_device_matches_reference(enc, case):
    sw, cs, nc, prec, (h, w), kind, script = case
    pix = image(zlib.crc32(_id(case).encode()), h, w, nc, prec, kind)
    p = params(sw, w, h, nc, cs, script)
    got = enc.encode_batch(p, pix[None])[0]
    assert hashlib.md5(got).hexdigest() == GOLDEN[_id(case)]
    if os.path.exists(REFLL):
        assert got == ref_encode(pix, sw, cs, script)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [12, 16])
def test_unaligned_16bit_input(enc, prec):
    # odd row pitch, image stride and base address: the C-ABI takes them unaligned
    import torch
    h, w = 17, 23
    imgs = np.stack([image(40 + i, h, w, 3, prec) for i in range(3)])
    sw = ["-revert", "-precision", str(prec), "-lossless", "7"]
    want = [ref_encode(imgs[i], sw, A.CS_RGB) for i in range(3)]
    pitch = w * 3 * 2 + 1
    stride = pitch * h + 3
    buf = np.zeros(1 + stride * 3, dtype=np.uint8)
    for i in range(3):
        for y in range(h):
            o = 1 + i * stride + y * pitch
            buf[o:o + w * 6] = np.frombuffer(imgs[i, y].tobytes(), dtype=np.uint8)
    p = mj.params_from_switches(sw, w, h, 3)
    enc.encode_batch_ptr(p, buf.ctypes.data + 1, False, pitch, stride, 3)
    assert [enc.get_output(i) for i in range(3)] == want
    t = torch.from_numpy(buf).cuda()
    enc.encode_batch_ptr(p, t.data_ptr() + 1, True, pitch, stride, 3)
    assert [enc.get_output(i) for i in range(3)] == want


@pytest.mark.gpu
def test_refused_restart_matches_reference(enc):
    pix = image(3, 9, 53, 3, 8)
    with pytest.raises(RuntimeError):
        ref_encode(pix, ["-revert", "-lossless", "4", "-restart", "40B"], A.CS_RGB)
    p = mj.params_from_switches(["-revert", "-lossless", "4", "-restart", "40B"], 53, 9, 3)
    with pytest.raises(mj.B200JpegError):
        enc.encode_batch(p, pix[None])


@pytest.mark.gpu
def test_device_memory_chunks_and_streams(enc):
    import torch
    h, w = 45, 61
    for prec, sw in ((16, ["-revert", "-precision", "16", "-lossless", "6,1", "-restart", "3"]), (8, ["-revert", "-lossless", "1"])):
        imgs = np.stack([image(10 + i, h, w, 3, prec) for i in range(7)])
        want = [ref_encode(imgs[i], sw, A.CS_RGB) for i in range(7)]
        p = mj.params_from_switches(sw, w, h, 3)
        enc.set_chunk_images(3)                                   # chunks of 3, 3, 1 on the two compute streams
        try:
            assert enc.encode_batch(p, imgs) == want
            t = torch.from_numpy(imgs.view(np.int16) if prec == 16 else imgs).cuda()
            enc.encode_batch_ptr(p, t.data_ptr(), True, imgs.strides[1], imgs.strides[0], 7)
            assert [enc.get_output(i) for i in range(7)] == want
        finally:
            enc.set_chunk_images(0)
        assert "lossless_diff" in enc.stage_times()


@pytest.mark.gpu
def test_streaming_entry_points(enc):
    for prec in (8, 12, 16):
        sw = ["-revert", "-precision", str(prec), "-lossless", "4,1"]
        pix = image(20 + prec, 14, 33, 3, prec)
        p = mj.params_from_switches(sw, 33, 14, 3)
        enc.start_compress(p)
        assert enc.write_scanlines(pix[:5]) == 5 and enc.write_scanlines(pix[5:]) == 9
        assert enc.finish_compress() == ref_encode(pix, sw, A.CS_RGB)


@pytest.mark.gpu
def test_live_random_shapes(enc):
    rng = np.random.default_rng(2026)
    switch_sets = [["-revert", "-lossless", "{psv},{pt}"], ["-revert", "-precision", "12", "-lossless", "{psv},{pt}", "-restart", "{r}"],
                   ["-revert", "-precision", "16", "-lossless", "{psv},{pt}"], ["-baseline", "-notrellis", "-lossless", "{psv},{pt}"]]
    for k in range(24):
        h, w = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        tmpl = switch_sets[k % len(switch_sets)]
        prec = 12 if "12" in tmpl else 16 if "16" in tmpl else 8
        sw = [s.format(psv=int(rng.integers(1, 8)), pt=int(rng.integers(0, prec)), r=int(rng.integers(1, 5))) for s in tmpl]
        nc = int(rng.choice([1, 3]))
        pix = image(k, h, w, nc, prec, "smooth" if k % 3 else "wide12" if prec > 8 else "alternating")
        want = ref_encode(pix, sw, A.CS_GRAYSCALE if nc == 1 else A.CS_RGB)
        p = mj.params_from_switches(sw, w, h, nc)
        assert enc.encode_batch(p, pix[None])[0] == want, sw


@pytest.mark.gpu
def test_raw_and_coefficient_inputs_refuse_lossless(enc):
    p = mj.params_from_switches(["-revert", "-lossless", "1"], 16, 16, 1)
    with pytest.raises(mj.B200JpegError):
        enc.encode_batch_raw(p, [np.zeros((1, 16, 16), np.uint8)])
    with pytest.raises(mj.B200JpegError):
        enc.encode_batch_coefs(p, [np.zeros((1, 2, 2, 64), np.int16)])


@pytest.mark.gpu
@pytest.mark.parametrize("switches,launches", [(["-baseline", "-quality", "75", "-sample", "2x2"], 17),
                                               (["-fastcrush", "-quality", "75", "-sample", "2x2"], 111),
                                               (["-quality", "75", "-sample", "2x2"], 1298)])
def test_lossy_launches_unchanged(switches, launches):
    # four bench-sized 3840x2160 images from host memory: the lossy paths launch what the commit before the lossless
    # encoder launched for the same call (counts measured with that commit's library on an H100)
    from mozjpeg_b200.synth import synth_image
    imgs = np.stack([synth_image(300 + i, 3840, 2160) for i in range(4)])
    e = mj.Encoder(0)
    try:
        e.encode_batch(mj.params_from_switches(switches, 3840, 2160, 3), imgs)
        assert e.kernel_launches() == launches
        assert "lossless_diff" not in e.stage_times()
    finally:
        e.close()
