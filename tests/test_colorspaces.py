"""CMYK, YCCK, YCbCr->grayscale and JCS_UNKNOWN encodes: the accept/refuse rules of jinit_color_converter
(jccolor.c:551-740) on the host, and the device path's files against the unmodified reference's
(tests/golden/colorspace_golden.json, tools/make_golden.py --colorspaces) through every entry point."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import colorspace_cases as CC

need_ref = pytest.mark.skipif(not CC.have_reference(), reason="build/librefcs.so not built (needs the reference build under oracle/_ref/)")
SHIM = os.path.join(CC.ROOT, "integration", "_build", "libjpeg_b200shim.so")
need_shim = pytest.mark.skipif(not (os.path.exists(SHIM) and os.path.exists(os.path.join(CC.REF, "tjbench"))),
                               reason="shim / reference tjbench not built (needs the reference build under oracle/_ref/)")


@pytest.fixture(scope="module")
def golden():
    return CC.load_golden()


def _params(c):
    import mozjpeg_b200 as mj
    in_cs, ic, jcs = CC.CONVERSIONS[c["conv"]]
    if c["kind"] == "tj":
        ss, opt, prog = c["tj"]
        return mj.tj3_params(c["w"], c["h"], 75, CC.TJ_SUBSAMP[ss], bool(opt), bool(prog), cmyk=True,
                             colorspace=None if CC.TJ_COLORSPACES[c["conv"]] < 0 else CC.CS_CMYK)
    return mj.params_from_switches(c["switches"], c["w"], c["h"], ic, in_cs, jcs)


# ------------------------------------------------------------------ host side (no GPU)
@need_ref
def test_reference_reproduces_the_recorded_files(golden):
    """The reference build in use writes the recorded bytes (pins the goldens and the driver's call order)."""
    for c in golden["cases"]:
        if c["w"] * c["h"] > 227 * 149:
            continue
        assert CC.md5(CC.reference_file(c)) == c["md5"], c["id"]


def test_oracle_restatement_reproduces_the_recorded_files(golden):
    """The CPU restatement (cmyk_ycck_convert in tests/colorspace_cases.py, the rest in oracle/jpeg_oracle.c) writes the
    reference's recorded bytes for every pixel and raw-data case; needs no reference build and no GPU."""
    import mozjpeg_b200 as mj
    bad = [c["id"] for c in golden["cases"] if CC.md5(CC.oracle_encode(_params(c), CC.case_image(c)).jpeg) != c["md5"]]
    for r in golden["raw"]:
        in_cs, jcs = CC.RAW_CONVERSIONS[r["conv"]]
        p = mj.params_from_switches(r["switches"], r["w"], r["h"], 4, in_cs, jcs)
        if CC.md5(CC.oracle_encode_raw(p, CC.raw_planes(r["seed"], p, 4))) != r["md5"]:
            bad.append(r["id"])
    assert not bad, bad


def test_cmyk_to_ycck_restatement_on_extremes():
    """White (C = M = Y = 0) is Y = MAXJSAMPLE with neutral chroma; full ink is Y = 0; K is never altered."""
    for prec, maxj in ((8, 255), (12, 4095)):
        dt = np.uint8 if prec == 8 else np.uint16
        px = np.array([[[0, 0, 0, 7], [maxj, maxj, maxj, maxj], [0, maxj, maxj, 0]]], dtype=dt)
        out = CC.cmyk_to_ycck(px, prec)
        c = (maxj + 1) // 2
        assert out[0, 0].tolist() == [maxj, c, c, 7] and out[0, 1].tolist() == [0, c, c, maxj]
        assert out[0, 2, 2] == maxj      # red: Cr at its maximum


def test_parameter_blocks_validate(golden):
    """Every recorded case's parameter block is accepted by b200jpeg_validate (on the device path)."""
    from mozjpeg_b200 import _abi as A
    lib = A.load()
    for c in golden["cases"]:
        p = _params(c)
        assert lib.b200jpeg_validate(C.byref(p)) == A.OK, (c["id"], lib.b200jpeg_last_error())


MATRIX_IN = [("unknown1", CC.CS_UNKNOWN, 1), ("unknown2", CC.CS_UNKNOWN, 2), ("unknown3", CC.CS_UNKNOWN, 3), ("unknown4", CC.CS_UNKNOWN, 4),
             ("gray", CC.CS_GRAYSCALE, 1), ("rgb", CC.CS_RGB, 3), ("bgrx", CC.CS_EXT_BGRX, 4), ("ycbcr", CC.CS_YCbCr, 3),
             ("cmyk", CC.CS_CMYK, 4), ("ycck", CC.CS_YCCK, 4)]
MATRIX_OUT = [("unknown", CC.CS_UNKNOWN), ("gray", CC.CS_GRAYSCALE), ("rgb", CC.CS_RGB), ("ycbcr", CC.CS_YCbCr), ("cmyk", CC.CS_CMYK), ("ycck", CC.CS_YCCK)]


@need_ref
@pytest.mark.parametrize("src", MATRIX_IN, ids=lambda s: s[0])
def test_accept_refuse_matrix(src):
    """b200jpeg_validate says OK exactly where the reference's jpeg_start_compress succeeds, and ERR_PARAM where it
    fails, for every (in_color_space, jpeg_color_space) pair."""
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    lib = A.load()
    _, in_cs, ic = src
    img = np.zeros((8, 8, ic), dtype=np.uint8)
    for name, jcs in MATRIX_OUT:
        try:
            CC.ref_encode(img, in_cs, ic, jcs, [])
            ref_ok = True
        except CC.RefError:
            ref_ok = False
        p = mj.params_from_switches([], 8, 8, ic, in_cs, jcs)
        rc = lib.b200jpeg_validate(C.byref(p))
        assert rc == (A.OK if ref_ok else A.ERR_PARAM), (src[0], name, rc, lib.b200jpeg_last_error())


def test_more_than_four_components_is_unsupported():
    from mozjpeg_b200 import _abi as A
    lib = A.load()
    p = A.Params()
    p.in_color_space, p.input_components, p.image_width, p.image_height = CC.CS_UNKNOWN, 4, 8, 8
    lib.b200jpeg_set_defaults(C.byref(p), A.PROFILE_MAX_COMPRESSION)
    assert p.num_components == 4 and lib.b200jpeg_validate(C.byref(p)) == A.OK
    p.input_components = 5
    assert lib.b200jpeg_set_colorspace(C.byref(p), CC.CS_UNKNOWN) == A.ERR_UNSUPPORTED
    p.input_components = 11
    assert lib.b200jpeg_set_colorspace(C.byref(p), CC.CS_UNKNOWN) == A.ERR_PARAM
    q = A.Params(); q.in_color_space, q.input_components, q.image_width, q.image_height = CC.CS_UNKNOWN, 4, 8, 8
    lib.b200jpeg_set_defaults(C.byref(q), A.PROFILE_MAX_COMPRESSION)
    q.num_components = q.input_components = 5
    assert lib.b200jpeg_validate(C.byref(q)) == A.ERR_UNSUPPORTED
    q.num_components = q.input_components = 11
    assert lib.b200jpeg_validate(C.byref(q)) == A.ERR_PARAM


def test_colorspace_defaults_follow_the_reference():
    """jpeg_set_colorspace (jcparam.c:624-648): component ids, sampling, Adobe marker."""
    from mozjpeg_b200 import _abi as A
    lib = A.load()
    p = A.Params(); p.in_color_space, p.input_components = CC.CS_CMYK, 4
    lib.b200jpeg_set_defaults(C.byref(p), A.PROFILE_MAX_COMPRESSION)
    assert p.jpeg_color_space == CC.CS_CMYK and p.write_Adobe_marker and not p.write_JFIF_header
    assert [p.comp_info[i].component_id for i in range(4)] == [0x43, 0x4D, 0x59, 0x4B]
    lib.b200jpeg_set_colorspace(C.byref(p), CC.CS_YCCK)
    assert [(c.component_id, c.h_samp_factor, c.v_samp_factor, c.quant_tbl_no) for c in p.comp_info] == [(1, 2, 2, 0), (2, 1, 1, 1), (3, 1, 1, 1), (4, 2, 2, 0)]
    p.input_components = 3
    lib.b200jpeg_set_colorspace(C.byref(p), CC.CS_UNKNOWN)
    assert p.num_components == 3 and not p.write_Adobe_marker
    assert [(p.comp_info[i].component_id, p.comp_info[i].h_samp_factor, p.comp_info[i].quant_tbl_no) for i in range(3)] == [(0, 1, 0), (1, 1, 0), (2, 1, 0)]


def test_jpegtran_mirror_refuses_grayscale_on_four_components(golden):
    """jpegtran -grayscale on a CMYK / YCCK source fails like the reference (JERR_CONVERSION_NOTIMPL), no file."""
    from mozjpeg_b200 import jpegtran as T
    for t in golden["transcode"]:
        if t["switches"] == ["-grayscale"]:
            assert "Unsupported color conversion" in t["error"]
    src = T.SourceInfo(); src.num_components = 4; src.jpeg_color_space = CC.CS_YCCK
    with pytest.raises(T.ConversionError):
        T.params_for_transcode(src, ["-grayscale"])


# ------------------------------------------------------------------ device path
@pytest.fixture(scope="module")
def enc():
    import mozjpeg_b200 as mj
    e = mj.Encoder(0)
    yield e
    e.close()


@pytest.mark.gpu
def test_every_golden_case_on_the_device(golden, enc):
    bad = []
    for c in golden["cases"]:
        out = enc.encode_batch(_params(c), CC.case_image(c)[None])[0]
        if CC.md5(out) != c["md5"]:
            bad.append((c["id"], len(out), c["size"]))
    assert not bad, bad


def _some_cases(golden, n_per_conv=3):
    seen = {}
    for c in golden["cases"]:
        if c["w"] == 227 and seen.get(c["conv"], 0) < n_per_conv:
            seen[c["conv"]] = seen.get(c["conv"], 0) + 1
            yield c


@pytest.mark.gpu
def test_device_resident_input_equals_host_input(golden, enc):
    import torch
    for c in _some_cases(golden):
        p, img = _params(c), CC.case_image(c)[None]
        host = enc.encode_batch(p, img)[0]
        t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
        torch.cuda.synchronize()
        es = t.element_size()
        enc.encode_batch_ptr(p, t.data_ptr(), True, t.stride(1) * es, t.stride(0) * es, 1)
        assert enc.get_output(0) == host and CC.md5(host) == c["md5"], c["id"]


@pytest.mark.gpu
def test_multi_chunk_batch_equals_single_encodes(golden, enc):
    import mozjpeg_b200 as mj
    for c in _some_cases(golden, 2):
        p = _params(c)
        in_cs, ic, _ = CC.CONVERSIONS[c["conv"]]
        prec = CC.precision_of(c.get("switches", []))
        imgs = np.stack([CC.cmyk_image(100 + i, c["w"], c["h"], ic, prec) for i in range(5)])
        singles = [enc.encode_batch(p, imgs[i:i + 1])[0] for i in range(5)]
        e2 = mj.Encoder(0)
        e2.set_chunk_images(2)                       # chunks of 2, 2 and 1 images
        assert e2.encode_batch(p, imgs) == singles, c["id"]
        assert e2.chunk_images() == 2
        e2.close()


@pytest.mark.gpu
def test_streaming_entry_points_produce_the_same_files(golden, enc):
    """b200jpeg_start_compress / write_scanlines / finish_compress, rows of W * input_components samples: uint8 rows,
    and uint16 rows (J12SAMPLE) for the 12-bit set."""
    import mozjpeg_b200 as mj
    twelve = [c for c in golden["cases"] if c["w"] == 227 and c["kind"] == "cjpeg" and CC.precision_of(c["switches"]) == 12]
    assert len(twelve) == len(CC.CONVERSIONS)
    for c in list(_some_cases(golden, 2)) + twelve:
        p, img = _params(c), CC.case_image(c)
        e2 = mj.Encoder(0)
        e2.start_compress(p)
        for y in range(0, img.shape[0], 7):
            e2.write_scanlines(img[y:y + 7])
        assert CC.md5(e2.finish_compress()) == c["md5"], c["id"]
        e2.close()


@pytest.mark.gpu
def test_raw_data_with_four_planes(golden, enc):
    import mozjpeg_b200 as mj
    for r in golden["raw"]:
        in_cs, jcs = CC.RAW_CONVERSIONS[r["conv"]]
        p = mj.params_from_switches(r["switches"], r["w"], r["h"], 4, in_cs, jcs)
        planes = CC.raw_planes(r["seed"], p, 4)
        out = enc.encode_batch_raw(p, [a[None] for a in planes])[0]
        assert CC.md5(out) == r["md5"], r["id"]


TAP_CASES = ["cmyk-ycck|-baseline -quality 75|227x149", "cmyk-ycck|-baseline -notrellis -quality 60 -sample 2x2,1x1,1x1,2x2|227x149",
             "cmyk-ycck|-quality 75|227x149", "cmyk-ycck|-precision 12 -notrellis -noovershoot -baseline|227x149",
             "cmyk-cmyk|-baseline -quality 75 -smooth 30|227x149", "unknown4|-dct float|227x149", "ycbcr-gray|-baseline -quality 75|227x149"]


@pytest.mark.gpu
@pytest.mark.parametrize("cid", TAP_CASES)
def test_stage_taps_match_oracle(golden, cid):
    """Raw DCT, plain-quantized and final coefficient planes of every component (YCCK's 10-block MCU included) and the
    trellis-phase Huffman tables equal the CPU restatement's, not just the file bytes."""
    import mozjpeg_b200 as mj
    c = next(x for x in golden["cases"] if x["id"] == cid)
    os.environ["B200JPEG_KEEP_PLAIN"] = "1"
    e = mj.Encoder(0)
    try:
        p = _params(c)
        in_cs, ic, _ = CC.CONVERSIONS[c["conv"]]
        imgs = np.stack([CC.cmyk_image(60 + i, c["w"], c["h"], ic, CC.precision_of(c["switches"])) for i in range(2)])
        out = e.encode_batch(p, imgs)
        for i in range(2):
            r = CC.oracle_encode(p, imgs[i], want_debug=True)
            d = r.dbg
            assert d["ncomp"] == p.num_components
            for ci in range(p.num_components):
                hib, wib = d["hib"][ci], d["wib"][ci]
                assert (e.debug_coefs(i, ci, 1)[:hib, :wib] == d["raw"][ci][:hib, :wib]).all(), ("raw", i, ci)
                assert (e.debug_coefs(i, ci, 2) == d["plain"][ci]).all(), ("plain", i, ci)
                assert (e.debug_coefs(i, ci, 0) == d["final"][ci]).all(), ("final", i, ci)
                if p.trellis_quant and p.num_scans == 0:       # (progressive trellis rounds keep the supplied DC table, no tap)
                    assert e.debug_huff(i, -1 - ci, False, p.comp_info[ci].dc_tbl_no) == d["trellis_dc"][ci]
                    assert e.debug_huff(i, -1 - ci, True, p.comp_info[ci].ac_tbl_no) == d["trellis_ac"][ci]
            assert out[i] == r.jpeg
    finally:
        e.close()
        os.environ.pop("B200JPEG_KEEP_PLAIN", None)


@need_ref
@pytest.mark.gpu
def test_coefficient_input_matches_jpegtran(golden, enc):
    """jpegtran's re-encode (default, -progressive, -optimize) of CMYK and YCCK sources through the host mirror and
    b200jpeg_encode_batch_coefs."""
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    for t in golden["transcode"]:
        if "md5" not in t or t["switches"] not in ([], ["-progressive"], ["-optimize"]):
            continue
        src = CC.tran_source(t["source"])
        assert CC.md5(src) == t["source_md5"]
        planes = O.ref_read_coefs(src)["coefs"]
        out = T.transcode(enc, [src], [pl[None] for pl in planes], t["switches"])[0]
        assert CC.md5(out) == t["md5"], t["id"]


# ------------------------------------------------------------------ the libjpeg boundary (reference binaries + shim)
def _ppm_cmyk(tmp_path):
    """tjbench reads a PPM and converts it to CMYK itself (-cmyk)."""
    img = CC.cmyk_image(11, 227, 149, 3)
    f = tmp_path / "img.ppm"
    f.write_bytes(b"P6\n227 149\n255\n" + img.tobytes())
    return f


def _tjbench(tmp_path, args, shim):
    d = tmp_path / ("shim" if shim else "plain")
    d.mkdir(exist_ok=True)
    ppm = _ppm_cmyk(d)
    env = dict(os.environ)
    if shim:
        env.update(LD_PRELOAD=SHIM, B200_SHIM_REQUIRE="1", B200_SHIM_VERBOSE="1")
    r = subprocess.run([os.path.join(CC.REF, "tjbench"), str(ppm), "75", "-cmyk", "-benchtime", "0.01", "-warmup", "0", "-componly", *args],
                       env=env, capture_output=True, text=True, timeout=600)
    jpgs = sorted(p for p in d.iterdir() if p.suffix == ".jpg")
    return r, jpgs


@need_shim
@pytest.mark.gpu
@pytest.mark.parametrize("args", [["-subsamp", "444"], ["-subsamp", "422"], ["-subsamp", "420"], ["-subsamp", "440"], ["-optimize"], ["-progressive"]],
                         ids=lambda a: "_".join(x.lstrip("-") for x in a))
def test_tjbench_cmyk_runs_on_the_device(args, tmp_path):
    r, got = _tjbench(tmp_path, args, True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "device path" in r.stderr, r.stderr
    r2, want = _tjbench(tmp_path, args, False)
    assert r2.returncode == 0 and got and [p.name for p in got] == [p.name for p in want]
    for a, b in zip(got, want):
        assert a.read_bytes() == b.read_bytes(), a.name


@need_shim
@pytest.mark.gpu
@pytest.mark.parametrize("src", CC.TRAN_SOURCES)
def test_reference_jpegtran_reencodes_four_components_on_the_device(src, golden, tmp_path):
    data = CC.tran_source(src)
    f = tmp_path / "src.jpg"
    f.write_bytes(data)
    env = dict(os.environ, LD_PRELOAD=SHIM, B200_SHIM_REQUIRE="1", B200_SHIM_VERBOSE="1")
    for t in golden["transcode"]:
        if t["source"] != src or "md5" not in t:
            continue
        r = subprocess.run([os.path.join(CC.REF, "jpegtran"), *t["switches"], str(f)], env=env, capture_output=True, timeout=600)
        assert r.returncode == 0, r.stderr.decode()
        assert b"device path (coefficients" in r.stderr, r.stderr.decode()
        assert CC.md5(r.stdout) == t["md5"], t["id"]
