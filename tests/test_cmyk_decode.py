"""Decompressing and recompressing 4-component (CMYK / YCCK) JPEG files on the device, opt-in through the `cmyk`
decompress option: the pixels the reference's decompressor makes (ycck_cmyk_convert / null_convert behind the
per-component IDCT and upsampling), the colour pairs it refuses, cjpeg's bytes from such files, and the unchanged
refusals without the option.  Sources and records: tests/cmyk_cases.py, tests/golden/cmyk_golden.json."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cmyk_cases as K
import decompress_options_cases as O
import recompress_cases as R

GOLD = K.golden()
CASE = {c["id"]: c for c in GOLD["cases"]}
CASES = K.cases()
SRC_MD5 = {s["id"]: s["md5"] for s in GOLD["sources"]}


def _info(jpeg):
    from mozjpeg_b200 import jpegtran as T
    return T.parse_source(jpeg)


@pytest.fixture(scope="module")
def enc():
    import mozjpeg_b200 as mj
    e = mj.Encoder(0)
    e.set_progressive_decode(True)
    yield e
    e.close()


# ------------------------------------------------------------------------------------------------------------ CPU
def test_cases_match_the_golden(built):
    assert [c[0] for c in CASES] == [c["id"] for c in GOLD["cases"]]
    for sid, m in SRC_MD5.items():
        assert K.md5(K.source(sid)) == m, sid
    assert _info(K.source("cmyk_dqt16")).sof == 0xC1
    assert _info(K.source("ycck_prog")).sof == 0xC2
    for sid in ("cmyk_444", "cmyk_420", "cmyk_k_sub"):
        assert _info(K.source(sid)).jpeg_color_space == K.CMYK, sid
    for sid in ("ycck_420", "ycck_libjpeg", "ycck_markers"):
        assert _info(K.source(sid)).jpeg_color_space == K.YCCK, sid


def test_numpy_ycck_cmyk_convert_matches_the_golden(built):
    # ycck_420 at 1/1 with ISLOW and fancy upsampling: Y and K full size, Cb and Cr h2v2_fancy_upsample
    src = K.source("ycck_420")
    planes = K.source_planes("ycck_420")
    info = _info(src)
    W, H = info.image_width, info.image_height
    s = [R.idct_plane(planes[c], list(info.comp_quant[c])) for c in range(4)]
    ycck = np.stack([s[0][:H, :W], R.upsample(s[1], 2, 2, W, H), R.upsample(s[2], 2, 2, W, H), s[3][:H, :W]], axis=-1).astype(np.uint8)
    assert K.md5(ycck) == CASE["ycck_420:1/1:int:fancy:ycck"]["pix_md5"]
    assert K.md5(K.ycck_to_cmyk(ycck)) == CASE["ycck_420:1/1:int:fancy:default"]["pix_md5"]
    # every (Y, Cb, Cr) against the scalar formula with the reference's range_limit
    g = np.stack(np.meshgrid(np.arange(256), np.arange(256), np.arange(0, 256, 5), indexing="ij"), -1).reshape(-1, 3)
    q = np.concatenate([g, np.full((len(g), 1), 9)], 1).astype(np.uint8)
    out = K.ycck_to_cmyk(q)
    for (y, cb, cr, _), o in zip(q[::997].astype(int), out[::997].astype(int)):
        r = y + ((91881 * (cr - 128) + 32768) >> 16)
        gg = y + ((-22554 * (cb - 128) - 46802 * (cr - 128) + 32768) >> 16)
        b = y + ((116130 * (cb - 128) + 32768) >> 16)
        assert list(o) == [min(max(255 - r, 0), 255), min(max(255 - gg, 0), 255), min(max(255 - b, 0), 255), 9]


def test_cmyk_to_rgb_and_the_ppm_framing(built):
    from mozjpeg_b200 import djpeg
    px = np.random.default_rng(3).integers(0, 256, (5, 7, 4), dtype=np.uint8)
    px[0, 0] = (255, 0, 128, 255); px[0, 1] = (1, 254, 127, 1)
    rgb = djpeg.cmyk_to_rgb(px)
    for y in range(5):
        for x in range(7):
            c, m, yy, k = (float(v) for v in px[y, x])
            assert tuple(rgb[y, x]) == tuple(int(v * k / 255.0 + 0.5) for v in (c, m, yy)), (y, x)
    assert djpeg.ppm_bytes(px) == b"P6\n7 5\n255\n" + rgb.tobytes()
    assert djpeg.parse([]) == dict(scale=(1, 1), dct="int", fancy=True, colorspace=None)


@pytest.mark.parametrize("i", range(len(CASES)))
def test_output_geometry_matches_the_reference(built, i):
    import mozjpeg_b200 as mj
    cid, sid, scale, dct, fancy, cs = CASES[i]
    rec = CASE[cid]
    w, h, ocs, nc = mj.decompress_output(_info(K.source(sid)), **K.opts(scale, dct, fancy, cs))
    assert [h, w, nc] == rec["shape"] and ocs == rec["out_color_space"], cid
    ow, oh, comps = O.plan(_info(K.source(sid)), scale, fancy)
    assert [[c[0], c[1], c[2]] for c in comps] == rec["components"], cid


def test_the_flag_changes_only_cmyk_and_ycck_output(built):
    import mozjpeg_b200 as mj
    for sid in ("cmyk_444", "ycck_420", "o_420", "o_gray"):
        info = _info(K.source(sid))
        for kw in ({}, dict(scale=(1, 2)), dict(scale=(1, 4), dct="fast", fancy=False)):
            assert mj.decompress_output(info, cmyk=True, **kw) == mj.decompress_output(info, cmyk=False, **kw), (sid, kw)
    assert mj.decompress_output(_info(K.source("ycck_420")), cmyk=True)[2:] == (K.CMYK, 4)
    for sid, cs in (("ycck_420", "cmyk"), ("ycck_420", "ycck"), ("cmyk_444", "cmyk")):
        info = _info(K.source(sid))
        with pytest.raises(mj.B200JpegError, match="not on the device path") as e:
            mj.decompress_output(info, colorspace=cs)
        assert e.value.code == mj._abi.ERR_UNSUPPORTED
        assert mj.decompress_output(info, colorspace=cs, cmyk=True)[2:] == ({"cmyk": K.CMYK, "ycck": K.YCCK}[cs], 4)
    assert mj._lib.b200jpeg_default_decompress_options().cmyk == 0 and mj.decompress_options().cmyk == 0 and mj.decompress_options(cmyk=True).cmyk == 1
    assert mj._abi.DecompressOptions(1, 1, 0, 1, -1, 0).cmyk == 0


@pytest.mark.parametrize("i", range(len(K.REFUSED_PAIRS)))
def test_refused_colour_pairs_carry_the_references_message(built, i):
    import mozjpeg_b200 as mj
    sid, cs = K.REFUSED_PAIRS[i]
    rec = GOLD["refused_pairs"][i]
    assert (rec["source"], rec["out_color_space"]) == (sid, cs)
    with pytest.raises(mj.B200JpegError, match=rec["message"]) as e:
        mj.decompress_output(_info(K.source(sid)), colorspace=cs, cmyk=True)
    assert e.value.code == mj._abi.ERR_PARAM
    with pytest.raises(mj.B200JpegError, match="RGB565"):
        mj.decompress_output(_info(K.source(sid)), colorspace="rgb565", cmyk=True)


@pytest.mark.parametrize("sid", ["cmyk_444", "ycck_420", "ycck_markers"])
def test_params_for_jpeg_input_of_a_cmyk_source(built, sid):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    src = K.source(sid)
    info = _info(src)
    for sw in (["-quality", "75"], ["-baseline", "-quality", "90"]):
        p = mj.params_for_jpeg_input(sw, src, cmyk=True)
        q = mj.params_from_switches(sw, info.image_width, info.image_height, 4, in_color_space=A.CS_CMYK)
        assert bytes(p) == bytes(q), (sid, sw)
        assert (p.in_color_space, p.input_components, p.jpeg_color_space, p.write_Adobe_marker) == (A.CS_CMYK, 4, A.CS_CMYK, 1)
        assert bytes(mj.params_for_jpeg_input(sw, src)) == bytes(p)
    markers = R.copied_markers(src, p)
    assert b"Adobe" not in markers
    if sid == "ycck_markers":
        assert markers.startswith(b"\xff\xfe") and b"\xff\xe2" in markers


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_every_golden_case_host_and_device_pointers(built, enc):
    import torch
    for cid, sid, scale, dct, fancy, cs in CASES:
        rec = CASE[cid]
        src = K.source(sid)
        kw = K.opts(scale, dct, fancy, cs)
        px = enc.decompress([src, src], **kw)
        assert list(px.shape[1:]) == rec["shape"] and K.md5(px[0]) == rec["pix_md5"] and (px[1] == px[0]).all(), cid
        h, w, nc = rec["shape"]
        pitch = (w * nc + 5) // 4 * 4 + 3                    # an odd pitch: no pixel of the second row is word-aligned
        t = torch.zeros((2, h, pitch), dtype=torch.uint8, device="cuda")
        enc.decompress_ptr([src, src], t.data_ptr(), pitch, h * pitch, **kw)
        got = t[:, :, :w * nc].cpu().numpy().reshape(2, h, w, nc)
        assert (got == px).all(), cid


@pytest.mark.gpu
def test_batches_equal_single_images_at_chunk_sizes_0_and_2(built, enc):
    files = [K.source(s) for s in ("ycck_420",) * 3] + [K.source("ycck_420")]
    kw = dict(scale=(1, 2), cmyk=True)
    one = enc.decompress([files[0]], **kw)[0]
    for chunk in (0, 2):
        enc.set_chunk_images(chunk)
        try:
            out = enc.decompress(files * 2, **kw)
        finally:
            enc.set_chunk_images(0)
        assert all((o == one).all() for o in out), chunk
    mixed = [K.source(s) for s in ("cmyk_444", "ycck_422", "ycck_w3", "cmyk_k_sub", "ycck_prog")]
    singles = [enc.decompress([f], cmyk=True)[0] for f in mixed]
    for chunk in (0, 2):
        enc.set_chunk_images(chunk)
        try:
            out = enc.decompress_mixed(mixed, [dict(cmyk=True)])[0]
        finally:
            enc.set_chunk_images(0)
        assert all((a == b).all() for a, b in zip(out, singles)), chunk


@pytest.mark.gpu
def test_a_rendition_ladder_equals_single_calls(built, enc):
    files = [K.source("ycck_libjpeg")] * 3
    rungs = [dict(cmyk=True), dict(scale=(1, 2), cmyk=True), dict(scale=(1, 4), cmyk=True, dct="fast")]
    outs = enc.decompress_renditions(files, rungs)
    for kw, o in zip(rungs, outs):
        assert (o == enc.decompress(files, **kw)).all(), kw
    # the same options twice share one pixel stage
    a, b = enc.decompress_renditions(files, [rungs[1], rungs[1]])
    assert (a == b).all()


@pytest.mark.gpu
def test_a_mixed_call_of_cmyk_ycck_ycbcr_and_gray_equals_per_file_calls(built, enc):
    from oracle import oracle as O2
    import mozjpeg_b200 as mj
    prog_rgb = O2.oracle_encode(mj.params_from_switches(["-progressive"], 90, 61, 3), O2.synth_image(4, 90, 61)).jpeg
    files = [K.source("cmyk_420"), O.source("o_420")[0], K.source("ycck_prog"), O.source("o_gray")[0], K.source("ycck_w5"),
             prog_rgb, K.source("cmyk_444"), K.source("ycck_444"), K.source("cmyk_444"), O.source("o_rgb")[0]]
    rungs = [dict(cmyk=True), dict(scale=(1, 2), cmyk=True, fancy=False), dict(scale=(3, 4), all_scales=True, cmyk=True)]
    out = enc.decompress_mixed(files, rungs)
    for r, kw in enumerate(rungs):
        for i, f in enumerate(files):
            assert (out[r][i] == enc.decompress([f], **kw)[0]).all(), (r, i)


@pytest.mark.gpu
def test_recompress_matches_the_references_bytes(built, enc):
    import mozjpeg_b200 as mj
    for rec in GOLD["recompress"]:
        src = K.source(rec["source"])
        p = mj.params_for_jpeg_input(rec["switches"], src, cmyk=True)
        out = enc.recompress(p, [src, src], cmyk=True)
        assert [len(out[0]), K.md5(out[0])] == [rec["size"], rec["md5"]] and out[1] == out[0], rec["id"]
        # recompress is encode_batch of the decompressed pixels, with the copied markers
        px = enc.decompress([src], cmyk=True)
        assert R.insert_markers(enc.encode_batch(p, px)[0], R.copied_markers(src, p)) == out[0], rec["id"]
    # the rendition and mixed forms
    src = K.source("ycck_420")
    sw = ["-quality", "75"]
    want = next(r for r in GOLD["recompress"] if r["id"] == "ycck_420:q75")["md5"]
    p = mj.params_for_jpeg_input(sw, src, cmyk=True)
    assert K.md5(enc.recompress_renditions([src], [(p, dict(cmyk=True))])[0][0]) == want
    got = enc.recompress_mixed([O.source("o_420")[0], src], [(sw, dict(cmyk=True))])[0]
    assert K.md5(got[1]) == want
    assert got[0] == enc.recompress(mj.params_for_jpeg_input(sw, O.source("o_420")[0]), [O.source("o_420")[0]])[0]


@pytest.mark.gpu
def test_the_cjpeg_and_djpeg_command_lines_take_cmyk_files(built, tmp_path):
    from mozjpeg_b200 import djpeg
    src = K.source("ycck_420")
    path = tmp_path / "in.jpg"
    path.write_bytes(src)
    env = dict(os.environ, PYTHONPATH=R.ROOT)
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.cjpeg", "-quality", "75", "-outfile", str(tmp_path / "o.jpg"), str(path)],
                       capture_output=True, env=env, cwd=R.ROOT)
    assert r.returncode == 0, r.stderr.decode()
    want = next(x for x in GOLD["recompress"] if x["id"] == "ycck_420:q75")
    assert K.md5((tmp_path / "o.jpg").read_bytes()) == want["md5"]
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.djpeg", "-outfile", str(tmp_path / "o.ppm"), str(path)], capture_output=True, env=env, cwd=R.ROOT)
    assert r.returncode == 0, r.stderr.decode()
    ppm = (tmp_path / "o.ppm").read_bytes()
    head = b"P6\n227 149\n255\n"
    assert ppm.startswith(head) and len(ppm) == len(head) + 227 * 149 * 3
    assert K.md5(ppm) == GOLD["djpeg_ppm"]["ycck_420"]


@pytest.mark.gpu
def test_without_the_flag_the_refusals_are_unchanged_and_launch_nothing(built, enc):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    good = O.source("o_420")[0]
    for sid in ("cmyk_444", "ycck_420", "ycck_prog"):
        f = K.source(sid)
        before = enc.kernel_launches()
        calls = [lambda: enc.decompress([f]), lambda: enc.decompress([f], scale=(1, 2)),
                 lambda: enc.recompress(mj.params_for_jpeg_input([], f), [f]),
                 lambda: enc.decompress_renditions([f], [{}, dict(scale=(1, 2))]),
                 lambda: enc.decompress_renditions([f], [dict(cmyk=True), dict(scale=(1, 2))])]
        for call in calls:
            with pytest.raises(A.B200JpegError) as e:
                call()
            assert e.value.code == A.ERR_UNSUPPORTED and str(e.value).endswith(
                "image 0: 4-component (CMYK / YCCK) source: only gray and 3-component files are decoded to pixels"), str(e.value)
        # a mixed call where one rung has cmyk and one does not names the image as before
        files = [good, good, f, good]
        for rungs in ([dict(cmyk=True), {}], [{}, dict(scale=(1, 2))]):
            with pytest.raises(A.B200JpegError) as e:
                enc.decompress_mixed(files, rungs)
            assert e.value.code == A.ERR_UNSUPPORTED and "image 2: 4-component (CMYK / YCCK) source" in str(e.value)
        assert enc.kernel_launches() == before, sid
        assert (enc.decompress([good]) == enc.decompress([good], cmyk=True)).all()
    # a factor of 3 stays refused with the option
    p = mj.tj3_params(48, 32, cmyk=True, subsamp="444")
    p.comp_info[0].h_samp_factor = 3
    from colorspace_cases import cmyk_image, oracle_encode
    f3 = oracle_encode(p, cmyk_image(1, 48, 32)).jpeg
    with pytest.raises(A.B200JpegError, match="image 0: 4-component"):
        enc.decompress_mixed([f3], [dict(cmyk=True)])
    # CMYK and YCCK coded files of one geometry are two conversions: refused in one single call, fine in a mixed call
    a, b = K.source("cmyk_420"), R.insert_markers(K.source("cmyk_420"), b"")
    c = K.source("ycck_420")
    with pytest.raises(A.B200JpegError, match="geometry"):
        enc.decompress([a, c], cmyk=True)
    m = enc.decompress_mixed([a, c, b], [dict(cmyk=True)])[0]
    assert (m[0] == enc.decompress([a], cmyk=True)[0]).all() and (m[1] == enc.decompress([c], cmyk=True)[0]).all()
