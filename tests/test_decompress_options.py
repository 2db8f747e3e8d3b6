"""Decompressing on the device with the decompress object's options (scale, dct_method, do_fancy_upsampling,
out_color_space): Encoder.decompress / recompress with options, b200jpeg_decompress_output_opts and the djpeg mirror,
against what the reference's decompressor produces with the same options (tests/golden/decompress_options_golden.json,
recorded by tools/make_golden.py --decompress-options; tests/refdecopt.c where the reference build exists)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import common  # noqa: F401,E402  (puts the repository root on sys.path)
import decompress_options_cases as O  # noqa: E402

GOLD = O.golden()
CASES = {c[0]: c for c in O.cases()}
PIX = {c["id"]: c for c in GOLD["cases"]}
IDS = list(CASES)

needs_reference = pytest.mark.skipif(not O.have_reference(), reason="the reference build (oracle/_ref, build/librefdecopt.so) is not here")


def _kw(cid):
    _, _, scale, dct, fancy, cs = CASES[cid]
    return dict(scale=scale, dct=dct, fancy=fancy, colorspace=cs)


def _info(jpeg):
    import mozjpeg_b200 as mj
    info = mj._abi.SourceInfo()
    mj._abi.check(mj._lib.b200jpeg_parse_source(jpeg, len(jpeg), C.byref(info)), "parse_source")
    return info


# ------------------------------------------------------------------------------------------------------------ CPU
def test_golden_covers_every_case():
    assert sorted(PIX) == sorted(IDS)


@pytest.mark.parametrize("cid", IDS)
def test_output_opts_and_plan_match_the_recorded_fields(built, cid):
    import mozjpeg_b200 as mj
    _, sid, scale, dct, fancy, cs = CASES[cid]
    jpeg, _ = O.source(sid)
    assert O.md5(jpeg) == PIX[cid]["src_md5"]
    info = _info(jpeg)
    w, h, ocs, nc = mj.decompress_output(info, **_kw(cid))
    shape = PIX[cid]["shape"]
    assert [h, w] + ([nc] if nc > 1 else []) == shape
    assert ocs == PIX[cid]["out_color_space"]
    ow, oh, comps = O.plan(info, scale, fancy)
    assert (ow, oh) == (w, h)
    assert [list(c[:3]) for c in comps] == PIX[cid]["components"]


@needs_reference
@pytest.mark.parametrize("cid", IDS[::7])
def test_reference_driver_reproduces_the_golden(cid):
    _, sid, scale, dct, fancy, cs = CASES[cid]
    px, info, msg = O.ref_decompress(O.source(sid)[0], O.opts_tuple(scale, dct, fancy, cs))
    assert px is not None, msg
    assert O.md5(px) == PIX[cid]["pix_md5"]


def test_default_options_and_validation(built):
    import mozjpeg_b200 as mj
    d = mj._lib.b200jpeg_default_decompress_options()
    assert (d.scale_num, d.scale_denom, d.dct_method, d.do_fancy_upsampling, d.out_color_space) == (1, 1, 0, 1, -1)
    info = _info(O.source("o_420")[0])
    assert mj.decompress_output(info, scale=(1, 5))[:2] == mj.decompress_output(info, scale=(1, 4))[:2] == (57, 38)
    for sc in O.REFUSED_SCALES:
        with pytest.raises(mj.B200JpegError, match="IDCT block size of %d" % O.block_size(*sc)):
            mj.decompress_output(info, scale=sc)
    for bad in ((0, 1), (1, 0)):
        with pytest.raises(mj.B200JpegError, match="must be positive"):
            mj.decompress_output(info, scale=bad)
    with pytest.raises(mj.B200JpegError, match="dct_method"):
        mj._abi.check(mj._lib.b200jpeg_decompress_output_opts(C.byref(info), C.byref(mj._abi.DecompressOptions(1, 1, 7, 1, -1)), None, None, None, None), "x")
    for cs in O.UNSUPPORTED_CS:
        with pytest.raises(mj.B200JpegError, match="not on the device path"):
            mj.decompress_output(info, colorspace=cs)
    with pytest.raises(ValueError):
        mj.decompress_options(dct="slow")


@pytest.mark.parametrize("i", range(len(O.REFUSED_PAIRS)))
def test_refused_colour_pairs_carry_the_references_message(built, i):
    import mozjpeg_b200 as mj
    sid, cs = O.REFUSED_PAIRS[i]
    rec = GOLD["refused_pairs"][i]
    assert (rec["source"], rec["out_color_space"]) == (sid, cs)
    with pytest.raises(mj.B200JpegError, match=rec["message"]):
        mj.decompress_output(_info(O.source(sid)[0]), colorspace=cs)


def test_djpeg_switches_and_ppm_framing(built):
    from mozjpeg_b200 import djpeg
    assert djpeg.parse(["-scale", "1/4", "-dct", "float", "-nosmooth", "-rgb"]) == dict(scale=(1, 4), dct="float", fancy=False, colorspace="rgb")
    assert djpeg.parse(["-fast"]) == dict(scale=(1, 1), dct="fast", fancy=False, colorspace=None)
    assert djpeg.parse(["-grayscale", "-pnm"]) == dict(scale=(1, 1), dct="int", fancy=True, colorspace="gray")
    for sw in (["-bmp"], ["-gif"], ["-targa"], ["-colors", "16"], ["-dither", "fs"], ["-crop", "8x8+0+0"], ["-skip", "1,2"], ["-rgb565"]):
        with pytest.raises(djpeg.NotOnDevice):
            djpeg.parse(sw)
    assert djpeg.ppm_bytes(np.zeros((2, 3, 3), np.uint8)) == b"P6\n3 2\n255\n" + bytes(18)
    assert djpeg.ppm_bytes(np.full((2, 3), 7, np.uint8)) == b"P5\n3 2\n255\n" + bytes([7] * 6)


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_every_golden_case_is_identical_to_the_reference(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    bad = []
    for cid in IDS:
        px = enc.decompress([O.source(CASES[cid][1])[0]], **_kw(cid))[0]
        if list(px.shape) != PIX[cid]["shape"] or O.md5(px) != PIX[cid]["pix_md5"]:
            bad.append(cid)
    enc.close()
    assert not bad, f"{len(bad)} of {len(IDS)} cases differ: {bad[:20]}"


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 2])
@pytest.mark.parametrize("kw", [dict(scale=(1, 2), dct="fast"), dict(scale=(1, 8), fancy=False, colorspace="bgrx"), dict(dct="float", colorspace="gray"),
                                dict(scale=(1, 4), colorspace="ycbcr")])
def test_batches_equal_single_images(built, chunk, kw):
    import mozjpeg_b200 as mj
    files = [O.source(s)[0] for s in ("s420", "q5", "q100", "sof1_dqt16", "restart_1")]     # one geometry, mixed tables
    enc = mj.Encoder(0)
    enc.set_chunk_images(chunk)
    batch = enc.decompress(files, **kw)
    for i, f in enumerate(files):
        assert np.array_equal(batch[i], enc.decompress([f], **kw)[0]), i
    enc.close()


@pytest.mark.gpu
def test_default_options_take_the_default_route(built):
    import mozjpeg_b200 as mj
    files = [O.source(s)[0] for s in ("s420", "q75")]
    enc = mj.Encoder(0)
    a = enc.decompress(files)
    b = enc.decompress(files, scale=(1, 1), dct="int", fancy=True, colorspace=None)
    c = enc.decompress(files, scale=(8, 8), colorspace="rgb")
    assert np.array_equal(a, b) and np.array_equal(a, c)
    p = mj.params_for_jpeg_input(["-quality", "80"], files[0])
    assert enc.recompress(p, files) == enc.recompress(p, files, scale=(2, 2))
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("sid,kw,sw", [("o_420", dict(scale=(1, 4)), ["-quality", "75", "-sample", "2x2"]),
                                        ("o_422", dict(scale=(1, 2), dct="float", fancy=False), ["-quality", "60"]),
                                        ("com_exif", dict(scale=(1, 8)), ["-revert"]),
                                        ("o_444", dict(scale=(1, 2), colorspace="bgrx"), ["-quality", "85"]),
                                        ("o_rgb", dict(scale=(1, 4), colorspace="gray"), [])])
def test_recompress_equals_encoding_the_decoded_rendition(built, sid, kw, sw):
    import mozjpeg_b200 as mj
    jpeg = O.source(sid)[0]
    p = mj.params_for_jpeg_input(sw, jpeg, **kw)
    enc = mj.Encoder(0)
    out = enc.recompress(p, [jpeg], **kw)[0]
    px = enc.decompress([jpeg], **kw)
    ref = enc.encode_batch(p, px if px.ndim == 4 else px[..., None])[0]
    import recompress_cases as R
    assert out == R.insert_markers(ref, R.copied_markers(jpeg, p))
    enc.close()


@pytest.mark.gpu
def test_refusals_name_the_image_and_the_encoder_recovers(built):
    import mozjpeg_b200 as mj
    from oracle import oracle as O2
    good = O.source("s420")[0]
    prog = O2.oracle_encode(mj.params_from_switches(["-progressive"], 200, 136), O2.synth_image(3, 200, 136)).jpeg
    enc = mj.Encoder(0)
    with pytest.raises(mj.B200JpegError, match="image 1: progressive"):
        enc.decompress([good, prog], scale=(1, 2))
    with pytest.raises(mj.B200JpegError, match="IDCT block size of 3"):
        enc.decompress([good], scale=(3, 8))
    with pytest.raises(mj.B200JpegError, match="Unsupported color conversion request"):
        enc.decompress([O.source("gray")[0]], colorspace="ycbcr")
    # a refused option set reads the same whether the pixels go to host or to device memory
    import ctypes as C
    import torch
    from mozjpeg_b200 import _abi as A
    _, ptrs, sizes = enc._files([good])
    o = mj.decompress_options(scale=(3, 8))
    host, dev = np.empty((136, 200, 3), dtype=np.uint8), torch.empty((136, 200, 3), dtype=torch.uint8, device="cuda")
    msgs = []
    for ptr, on_device in ((host.ctypes.data, 0), (dev.data_ptr(), 1)):
        with pytest.raises(mj.B200JpegError) as e:
            A.check(A.load().b200jpeg_decompress_batch_opts(enc._h, C.byref(o), ptrs, sizes, 1, ptr, on_device, 600, 600 * 136), "decompress_batch_opts")
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and "IDCT block size of 3" in msgs[0], msgs
    want = PIX["o_420:1/2:int:fancy:default"]
    assert O.md5(enc.decompress([O.source("o_420")[0]], scale=(1, 2))[0]) == want["pix_md5"]
    enc.close()


@pytest.mark.gpu
@needs_reference
def test_djpeg_cli_matches_the_reference(built, tmp_path):
    from mozjpeg_b200 import djpeg
    jpeg = O.source("o_420")[0]
    src = tmp_path / "in.jpg"
    src.write_bytes(jpeg)
    for sw, opts in ((["-scale", "1/4"], (1, 4, 0, 1, -1)), (["-fast", "-grayscale"], (1, 1, 1, 0, 1)), (["-scale", "1/2", "-dct", "float", "-nosmooth"], (1, 2, 2, 0, -1))):
        out = tmp_path / "out.pnm"
        r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.djpeg", *sw, "-outfile", str(out), str(src)], capture_output=True, cwd=O.ROOT)
        assert r.returncode == 0, r.stderr
        px, _, _ = O.ref_decompress(jpeg, opts)
        assert out.read_bytes() == djpeg.ppm_bytes(px)
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.djpeg", "-bmp", str(src)], capture_output=True, cwd=O.ROOT)
    assert r.returncode == 1 and b"not on the device path" in r.stderr
