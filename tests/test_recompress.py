"""Recompressing JPEG files on the device (cjpeg's JPEG input): Encoder.decompress / Encoder.recompress and the cjpeg
mirror against what the reference's decompressor and cjpeg produce (tests/golden/recompress_golden.json, recorded by
tools/make_golden.py --recompress), and the numpy restatement of the decompressor against both."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import common  # noqa: F401,E402  (puts the repository root on sys.path)
import decode_cases as D  # noqa: E402
import recompress_cases as R  # noqa: E402

GOLD = R.golden()
PIX = {c["id"]: c for c in GOLD["cases"]}
REC = GOLD["recompress"]
REC_IDS = [r["source"] + ":" + ("_".join(s.lstrip("-") for s in r["switches"]) or "default") for r in REC]

needs_reference = pytest.mark.skipif(not R.have_reference(), reason="the reference build (oracle/_ref, build/librefdec.so) is not here")


# ------------------------------------------------------------------------------------------------------------ CPU
def test_golden_covers_every_case():
    assert sorted(PIX) == sorted(R.all_ids())
    assert [(r["source"], r["switches"]) for r in REC] == [(s, sw) for s, sw in R.RECOMPRESS]


@pytest.mark.parametrize("sid", R.all_ids())
def test_numpy_restatement_reproduces_the_recorded_pixels(built, sid):
    jpeg, planes = R.source(sid)
    assert R.md5(jpeg) == PIX[sid]["src_md5"]
    px = R.decode_pixels(jpeg, planes)
    assert list(px.shape) == PIX[sid]["shape"]
    assert R.md5(px) == PIX[sid]["pix_md5"]


@needs_reference
@pytest.mark.parametrize("sid", R.all_ids())
def test_reference_decompressor_reproduces_the_recorded_pixels(built, sid):
    jpeg, planes = R.source(sid)
    px, info = R.ref_decompress(jpeg)
    assert R.md5(px) == PIX[sid]["pix_md5"] and info[5] == 0
    assert np.array_equal(px, R.decode_pixels(jpeg, planes))


@needs_reference
@pytest.mark.parametrize("k", range(len(REC)), ids=REC_IDS)
def test_reference_cjpeg_reproduces_the_recorded_files(built, k):
    out = R.ref_cjpeg(R.source(REC[k]["source"])[0], REC[k]["switches"])
    assert (R.md5(out), len(out)) == (REC[k]["md5"], REC[k]["size"])


@pytest.mark.parametrize("sid", ["gray", "s420", "s444", "rgb"])
def test_decompress_output_is_the_reference_out_color_space(built, sid):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    jpeg, _ = R.source(sid)
    w, h, cs, nc = mj.decompress_output(T.parse_source(jpeg))
    shape = PIX[sid]["shape"]
    assert [h, w] == shape[:2] and nc == (shape[2] if len(shape) == 3 else 1)
    assert cs == PIX[sid]["out_color_space"]                  # JCS_GRAYSCALE = 1, JCS_RGB = 2, like B200JPEG_CS_*
    if R.have_reference():
        info = R.ref_decompress(jpeg, header_only=True)[1]
        assert [w, h, nc, cs] == info[:4]


def test_decompress_output_of_a_four_component_source(built):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T, _abi as A
    assert mj.decompress_output(T.parse_source(D.extra_source("ycck")))[2:] == (A.CS_CMYK, 4)


@pytest.mark.parametrize("k", range(len(REC)), ids=REC_IDS)
def test_cjpeg_parameter_block_for_a_jpeg_input(built, k):
    """the mirror's block for a JPEG input is the one for a PPM of the decoded pixels, and the oracle's file for it,
    with the source's markers copied as cjpeg does, is the reference cjpeg's"""
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    jpeg, planes = R.source(REC[k]["source"])
    px = R.decode_pixels(jpeg, planes)
    p = mj.params_for_jpeg_input(REC[k]["switches"], jpeg)
    q = mj.params_from_switches(REC[k]["switches"], px.shape[1], px.shape[0], 1 if px.ndim == 2 else 3)
    assert bytes(p) == bytes(q)
    out = R.insert_markers(O.oracle_encode(p, px).jpeg, R.copied_markers(jpeg, p))
    assert (R.md5(out), len(out)) == (REC[k]["md5"], REC[k]["size"])


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("sid", R.all_ids())
def test_device_decompress_equals_the_reference(encoder, sid):
    jpeg, planes = R.source(sid)
    px = encoder.decompress([jpeg])[0]
    assert np.array_equal(px, R.decode_pixels(jpeg, planes))
    assert R.md5(px) == PIX[sid]["pix_md5"]


@pytest.mark.gpu
def test_decompress_stage_times(encoder):
    encoder.decompress([R.source("s420")[0]])
    st = encoder.stage_times()
    assert {"dec_h2d", "dec_sync", "dec_write", "dec_dc", "idct", "upsample_color"} <= set(st) and st["idct"] > 0 and st["upsample_color"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("sid", ["ragged_420", "ragged_422", "ragged_440", "ragged_444", "gray", "w5_420"])
def test_decompress_into_device_memory_with_an_odd_pitch(encoder, sid):
    """pixels left on the device, rows 1 byte further apart than a multiple of 4: the byte-store path"""
    import torch
    jpeg, planes = R.source(sid)
    want = R.decode_pixels(jpeg, planes)
    h, w = want.shape[:2]
    nc = 1 if want.ndim == 2 else 3
    for pad in (1, 4):
        pitch = (w * nc + 3) // 4 * 4 + pad
        buf = torch.full((2, h, pitch), 0xA5, dtype=torch.uint8, device="cuda")
        encoder.decompress_ptr([jpeg, jpeg], buf.data_ptr(), pitch, h * pitch)
        torch.cuda.synchronize()
        got = buf.cpu().numpy()
        for i in range(2):
            assert np.array_equal(got[i, :, :w * nc].reshape(want.shape), want)
        assert (got[:, :, w * nc:] == 0xA5).all()                  # nothing written between the rows


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(REC)), ids=REC_IDS)
def test_device_recompress_equals_the_reference_cjpeg(encoder, k):
    import mozjpeg_b200 as mj
    jpeg, _ = R.source(REC[k]["source"])
    out = encoder.recompress(mj.params_for_jpeg_input(REC[k]["switches"], jpeg), [jpeg])[0]
    assert (R.md5(out), len(out)) == (REC[k]["md5"], REC[k]["size"])


@pytest.mark.gpu
def test_copied_markers_keep_their_order_and_are_not_duplicated(encoder):
    import mozjpeg_b200 as mj
    jpeg, _ = R.source("com_exif")
    out = encoder.recompress(mj.params_for_jpeg_input(["-quality", "60"], jpeg), [jpeg])[0]
    assert out[2:4] == b"\xff\xe0" and out[20:20 + len(R.COM + R.EXIF)] == R.COM + R.EXIF and out.count(b"JFIF\0") == 1
    rgb, _ = R.source("rgb")
    assert rgb.count(b"Adobe") == 1
    assert encoder.recompress(mj.params_for_jpeg_input(["-revert", "-rgb"], rgb), [rgb])[0].count(b"Adobe") == 1
    # a YCbCr destination writes no Adobe marker of its own, so the source's is copied
    assert encoder.recompress(mj.params_for_jpeg_input(["-quality", "60"], rgb), [rgb])[0].count(b"Adobe") == 1
    # no marker of an earlier batch reaches a later pixel encode
    from oracle import oracle as O
    p = mj.params_from_switches(["-quality", "75"], 64, 48, 3)
    im = O.synth_image(1, 64, 48)
    assert encoder.encode_batch(p, im[None])[0] == O.oracle_encode(p, im).jpeg


@pytest.mark.gpu
def test_cjpeg_mirror_takes_a_jpeg_input(encoder, tmp_path):
    import importlib
    import mozjpeg_b200 as mj
    CJ = importlib.import_module("mozjpeg_b200.cjpeg")          # the package's cjpeg attribute is the function
    r = next(r for r in REC if r["source"] == "s420" and r["switches"] == ["-quality", "60"])
    jpeg, _ = R.source("s420")
    src, dst = tmp_path / "in.jpg", tmp_path / "out.jpg"
    src.write_bytes(jpeg)
    assert CJ.main(["-quality", "60", "-outfile", str(dst), str(src)]) == 0
    assert R.md5(dst.read_bytes()) == r["md5"]
    assert R.md5(mj.cjpeg(["-quality", "60"], jpeg, encoder)) == r["md5"]


MIXED = ["s420", "q5", "q100", "sof1_dqt16", "restart_1", "multi_scan", "q75"]      # one geometry; tables, restarts, scans differ


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 2])
def test_mixed_batch_equals_the_single_image_results(encoder, chunk):
    import mozjpeg_b200 as mj
    files = [R.source(s)[0] for s in MIXED]
    sw = ["-baseline", "-quality", "75", "-sample", "2x2"]
    p = mj.params_for_jpeg_input(sw, files[0])
    singles = [encoder.recompress(p, [f])[0] for f in files]
    encoder.set_chunk_images(chunk)
    try:
        px = encoder.decompress(files)
        for i, s in enumerate(MIXED):
            assert R.md5(px[i]) == PIX[s]["pix_md5"], s
        assert encoder.recompress(p, files) == singles
        assert encoder.recompress(p, files) == encoder.encode_batch(p, px)
    finally:
        encoder.set_chunk_images(0)
    for sw in ([], ["-revert", "-progressive", "-restart", "2"]):
        p = mj.params_for_jpeg_input(sw, files[0])
        assert encoder.recompress(p, files) == encoder.encode_batch(p, px)


def _refused(encoder, files, code, image, word, p=None):
    from mozjpeg_b200 import _abi as A
    with pytest.raises(A.B200JpegError) as ei:
        encoder.recompress(p, files) if p is not None else encoder.decompress(files)
    assert ei.value.code == code and f"image {image}:" in str(ei.value) and word in str(ei.value), str(ei.value)


@pytest.mark.gpu
def test_refusals_name_the_image_and_the_encoder_recovers(encoder):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    good, planes = R.source("s420")
    _refused(encoder, [D.extra_source("baseline12")], A.ERR_UNSUPPORTED, 0, "12-bit")
    _refused(encoder, [D.extra_source("cmyk")], A.ERR_UNSUPPORTED, 0, "4-component")
    s32 = D.source(next(c for c in D.CASES if c[0] == "sample_3x2"))[0]
    _refused(encoder, [good, s32], A.ERR_UNSUPPORTED, 1, "sampling")
    prog = O.oracle_encode(mj.params_from_switches(["-progressive", "-revert"], 200, 136, 3), D.pixels(3, 200, 136)).jpeg
    _refused(encoder, [good, good, prog], A.ERR_UNSUPPORTED, 2, "progressive")
    sc = T.parse_source(good).scans[0]
    truncated = good[:sc.data_offset + sc.data_size // 2]
    encoder.set_chunk_images(2)
    try:
        _refused(encoder, [good, good, good, truncated], A.ERR_BAD_SOURCE, 3, "corrupt")
        _refused(encoder, [good, good, good, truncated], A.ERR_BAD_SOURCE, 3, "corrupt", mj.params_for_jpeg_input([], good))
    finally:
        encoder.set_chunk_images(0)
    other = R.source("ragged_420")[0]
    _refused(encoder, [good, other], A.ERR_PARAM, 1, "geometry")
    with pytest.raises(A.B200JpegError) as ei:                  # a parameter block for another size
        encoder.recompress(mj.params_for_jpeg_input([], other), [good])
    assert ei.value.code == A.ERR_PARAM
    assert np.array_equal(encoder.decompress([good])[0], R.decode_pixels(good, planes))
    p = mj.params_from_switches(["-quality", "75"], 64, 48, 3)
    im = O.synth_image(1, 64, 48)
    assert encoder.encode_batch(p, im[None])[0] == O.oracle_encode(p, im).jpeg
