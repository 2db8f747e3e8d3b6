"""Rendition ladders: Encoder.decompress_renditions / recompress_renditions (b200jpeg_decompress_renditions /
b200jpeg_recompress_renditions) decode each source once and make several renditions of it.  Every rung must be byte
for byte what the single-rendition call makes with the same options (and params), the pixels also what the reference's
decompressor makes (tests/golden/decompress_options_golden.json), and the files what the reference's cjpeg makes where
the reference build exists."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import common  # noqa: F401,E402  (puts the repository root on sys.path)
import decompress_options_cases as O  # noqa: E402
import recompress_cases as R  # noqa: E402

PIX = {c["id"]: c for c in O.golden()["cases"]}

needs_reference = pytest.mark.skipif(not (O.have_reference() and R.have_reference()),
                                     reason="the reference build (oracle/_ref, build/librefdecopt.so, build/librefdec.so) is not here")

# one ladder that mixes scales, IDCT methods, fancy upsampling, output colour spaces and baseline / progressive params:
# (cjpeg switches, decompress options)
LADDER = [
    (["-baseline", "-quality", "80"], {}),
    (["-quality", "75"], dict(scale=(1, 2), dct="fast")),
    (["-revert", "-progressive", "-quality", "70"], dict(scale=(1, 4), dct="float", fancy=False, colorspace="bgrx")),
    (["-baseline", "-quality", "60"], dict(scale=(1, 8), colorspace="gray")),
    (["-quality", "85"], dict(dct="float", fancy=False)),
    (["-baseline", "-quality", "90"], dict(scale=(1, 2), colorspace="xrgb")),
]


def _rungs(jpeg, ladder=LADDER):
    import mozjpeg_b200 as mj
    return [(mj.params_for_jpeg_input(sw, jpeg, **kw), kw) for sw, kw in ladder]


def _info(jpeg):
    import mozjpeg_b200 as mj
    info = mj._abi.SourceInfo()
    mj._abi.check(mj._lib.b200jpeg_parse_source(jpeg, len(jpeg), C.byref(info)), "parse_source")
    return info


def _err(fn):
    import mozjpeg_b200 as mj
    with pytest.raises(mj.B200JpegError) as e:
        fn()
    return e.value


def _message(e):
    """the library's message of a B200JpegError, without the Python call site in front of it"""
    return str(e).split(": error ", 1)[1].split(": ", 1)[1]


def _stage_names(enc):
    import mozjpeg_b200 as mj
    names = (C.c_char_p * 64)(); ms = (C.c_float * 64)()
    k = mj._lib.b200jpeg_last_stage_times(enc._h, names, ms, 64)
    return [names[i].decode() for i in range(k)]


def _no_encoder():
    """an Encoder whose methods can run up to their first library call without a device"""
    import mozjpeg_b200 as mj
    return mj.Encoder.__new__(mj.Encoder)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_python_arguments_are_checked_before_any_call(built):
    import mozjpeg_b200 as mj
    enc = _no_encoder()
    jpeg = O.source("o_420")[0]
    p = mj.params_for_jpeg_input([], jpeg)
    for bad in ([], [dict(scale=(1, 2)), dict(sclae=(1, 2))], [dict(quality=80)], [(1, 2)]):
        with pytest.raises(ValueError):
            enc.decompress_renditions([jpeg], bad)
        with pytest.raises(ValueError):
            enc.decompress_renditions_ptr([jpeg], bad, [0] * len(bad), [0] * len(bad), [0] * len(bad))
    with pytest.raises(ValueError, match="unknown option 'sclae'"):
        enc.decompress_renditions([jpeg], [{}, dict(sclae=(1, 2))])
    with pytest.raises(ValueError, match="3 pointers"):
        enc.decompress_renditions_ptr([jpeg], [{}, {}, {}], [0, 0], [0, 0], [0, 0])
    for bad in ([], [(p, dict(fast=True))], [p], [(p,)], [({}, p)], [(p, {}, {})], [(p, dict(dct="slow"))]):
        with pytest.raises(ValueError):
            enc.recompress_renditions([jpeg], bad)


@pytest.mark.parametrize("sid", [lay[0] for lay in O.LAYOUTS])
def test_output_opts_give_each_rungs_geometry(built, sid):
    import mozjpeg_b200 as mj
    jpeg = O.source(sid)[0]
    info = _info(jpeg)
    for sw, kw in LADDER:
        w, h, cs, nc = mj.decompress_output(info, **kw)
        ow, oh, _ = O.plan(info, kw.get("scale", (1, 1)), kw.get("fancy", True))
        assert (w, h) == (ow, oh)
        p = mj.params_for_jpeg_input(sw, jpeg, **kw)
        assert (p.image_width, p.image_height, p.input_components, p.in_color_space) == (w, h, nc, cs)
        cid = O.case_id(sid, kw.get("scale", (1, 1)), kw.get("dct", "int"), kw.get("fancy", True), kw.get("colorspace"))
        if cid in PIX:
            assert PIX[cid]["shape"] == [h, w] + ([nc] if nc > 1 else [])


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("sid", [lay[0] for lay in O.LAYOUTS])
def test_every_layout_equals_the_single_calls(encoder, sid):
    jpeg = O.source(sid)[0]
    rungs = _rungs(jpeg)
    opts = [kw for _, kw in rungs]
    pixels = encoder.decompress_renditions([jpeg], opts)
    pinned = 0
    for r, kw in enumerate(opts):
        single = encoder.decompress([jpeg], **kw)
        assert pixels[r].shape == single.shape and np.array_equal(pixels[r], single), r
        cid = O.case_id(sid, kw.get("scale", (1, 1)), kw.get("dct", "int"), kw.get("fancy", True), kw.get("colorspace"))
        if cid in PIX:
            assert O.md5(pixels[r][0]) == PIX[cid]["pix_md5"], cid
            pinned += 1
    assert pinned >= 3
    files = encoder.recompress_renditions([jpeg], rungs)
    for r, (p, kw) in enumerate(rungs):
        assert files[r] == encoder.recompress(p, [jpeg], **kw), r


@pytest.mark.gpu
@needs_reference
@pytest.mark.parametrize("sid", ["o_420", "o_422", "o_gray"])
def test_rungs_equal_the_reference(encoder, sid):
    from mozjpeg_b200 import djpeg
    jpeg = O.source(sid)[0]
    ladder = [(["-quality", "80", "-sample", "2x2"], {}), (["-quality", "75"], dict(scale=(1, 4))),
              (["-baseline", "-quality", "70"], dict(scale=(1, 2), dct="float", fancy=False)), (["-quality", "70"], dict(scale=(1, 8)))]
    rungs = _rungs(jpeg, ladder)
    files = encoder.recompress_renditions([jpeg], rungs)
    assert files[0][0] == R.ref_cjpeg(jpeg, ladder[0][0])
    for r, (sw, kw) in enumerate(ladder[1:], 1):
        px, _, msg = O.ref_decompress(jpeg, O.opts_tuple(kw["scale"], kw.get("dct", "int"), kw.get("fancy", True), None))
        assert px is not None, msg
        # the reference's cjpeg reads the PPM of the scaled decode; the device copies the source's COM / APPn segments
        ref = R.ref_cjpeg(djpeg.ppm_bytes(px), sw)
        assert files[r][0] == R.insert_markers(ref, R.copied_markers(jpeg, rungs[r][0])), r


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 1, 2])
def test_batches_equal_single_image_ladders(encoder, chunk):
    import torch
    files = [O.source(s)[0] for s in ("s420", "q5", "q100", "sof1_dqt16", "restart_1")]     # one geometry, mixed tables and restarts
    rungs = _rungs(files[0])
    opts = [kw for _, kw in rungs]
    encoder.set_chunk_images(chunk)
    try:
        out = encoder.recompress_renditions(files, rungs)
        assert len(out) == len(rungs) and all(len(o) == len(files) for o in out)
        px = encoder.decompress_renditions(files, opts)
        for i, f in enumerate(files):
            single = encoder.recompress_renditions([f], rungs)
            single_px = encoder.decompress_renditions([f], opts)
            for r in range(len(rungs)):
                assert out[r][i] == single[r][0], (r, i)
                assert np.array_equal(px[r][i], single_px[r][0]), (r, i)
        # device pointers: each rung into a torch tensor with a padded row pitch
        bufs, pitch, stride = [], [], []
        for r in range(len(rungs)):
            a = px[r] if px[r].ndim == 4 else px[r][..., None]
            n, h, w, c = a.shape
            bufs.append(torch.full((n, h, w * c + 5), 7, dtype=torch.uint8, device="cuda"))
            pitch.append(w * c + 5); stride.append(h * (w * c + 5))
        torch.cuda.synchronize()
        encoder.decompress_renditions_ptr(files, opts, [b.data_ptr() for b in bufs], pitch, stride)
        for r in range(len(rungs)):
            a = px[r] if px[r].ndim == 4 else px[r][..., None]
            n, h, w, c = a.shape
            got = bufs[r].cpu().numpy()
            assert np.array_equal(got[:, :, :w * c].reshape(a.shape), a), r
            assert (got[:, :, w * c:] == 7).all(), r
    finally:
        encoder.set_chunk_images(0)


@pytest.mark.gpu
def test_duplicate_rungs_equal_their_single_calls(encoder):
    import torch
    files = [O.source(s)[0] for s in ("s420", "q75")]
    half = dict(scale=(1, 2))
    ladder = [(["-quality", "80"], half), (["-quality", "50", "-baseline"], half), (["-quality", "80"], half), ([], {}),
              (["-quality", "65"], dict(scale=(1, 2), dct="int", fancy=True, colorspace=None)), ([], {})]
    rungs = _rungs(files[0], ladder)
    out = encoder.recompress_renditions(files, rungs)
    for r, (p, kw) in enumerate(rungs):
        assert out[r] == encoder.recompress(p, files, **kw), r
    assert out[0] == out[2] and out[3] == out[5] and out[0] != out[1]
    opts = [kw for _, kw in ladder]
    px = encoder.decompress_renditions(files, opts)
    for r, kw in enumerate(opts):
        assert np.array_equal(px[r], encoder.decompress(files, **kw)), r
    bufs = [torch.zeros(a.shape, dtype=torch.uint8, device="cuda") for a in px]
    torch.cuda.synchronize()
    encoder.decompress_renditions_ptr(files, opts, [b.data_ptr() for b in bufs], [b.stride(1) for b in bufs], [b.stride(0) for b in bufs])
    for r in range(len(opts)):
        assert np.array_equal(bufs[r].cpu().numpy(), px[r]), r


@pytest.fixture(scope="module")
def progressive_sources(built):
    """mozjpeg's default profile (progressive, scan search), without and with restarts, written by the CPU oracle.  The
    restarts are counted in MCUs: with -restart in rows the scan search writes one DRI for scans whose intervals differ,
    and the device decode refuses such files (a restart segment count that does not match the DRI)."""
    import mozjpeg_b200 as mj
    from oracle import oracle as OR
    out = {}
    for name, sw in (("default", []), ("restart_2B", ["-restart", "2B"])):
        p = mj.params_from_switches(sw, 120, 88)
        out[name] = [OR.oracle_encode(p, OR.synth_image(70 + k, 120, 88)).jpeg for k in range(3)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["default", "restart_2B"])
def test_progressive_sources(encoder, progressive_sources, name):
    files = progressive_sources[name]
    assert all(f[:2] == b"\xff\xd8" and b"\xff\xc2" in f for f in files)
    rungs = _rungs(files[0])
    e = _err(lambda: encoder.recompress_renditions(files, rungs))
    single = _err(lambda: encoder.recompress(rungs[1][0], files, **rungs[1][1]))
    assert _message(e) == _message(single) and "image 0: progressive" in _message(e)
    encoder.set_progressive_decode(True)
    try:
        out = encoder.recompress_renditions(files, rungs)
        for r, (p, kw) in enumerate(rungs):
            assert out[r] == encoder.recompress(p, files, **kw), r
        px = encoder.decompress_renditions(files, [kw for _, kw in rungs])
        for r, (_, kw) in enumerate(rungs):
            assert np.array_equal(px[r], encoder.decompress(files, **kw)), r
        assert "dec_ac_refine" in _stage_names(encoder)
    finally:
        encoder.set_progressive_decode(False)


@pytest.mark.gpu
def test_the_decode_runs_once(encoder):
    files = [O.source(s)[0] for s in ("s420", "q5", "restart_1")]
    rungs = _rungs(files[0], [(["-quality", "80"], dict(scale=(1, 2))), (["-baseline", "-quality", "60"], dict(scale=(1, 4), dct="fast"))])
    encoder.set_chunk_images(len(files))
    try:
        encoder.recompress_renditions(files, rungs)                   # warm: buffers sized, tables cached
        k0 = encoder.kernel_launches()
        for p, kw in rungs:
            encoder.recompress(p, files, **kw)
        k1 = encoder.kernel_launches()
        encoder.recompress_renditions(files, rungs)
        names = _stage_names(encoder)
        k2 = encoder.kernel_launches()
        encoder.read_coefficients(files)
        k3 = encoder.kernel_launches()
    finally:
        encoder.set_chunk_images(0)
    assert k3 > k2
    assert (k1 - k0) - (k2 - k1) == k3 - k2
    dec = [s for s in names if s.startswith("dec_")]
    assert dec and len(dec) == len(set(dec))
    assert names.count("idct") == 1 and names.count("upsample_color") == 1
    assert len(names) == len(set(names))


@pytest.mark.gpu
def test_refusals(encoder):
    from mozjpeg_b200 import _abi as A
    good = O.source("s420")[0]
    files = [good, O.source("q75")[0]]
    rungs = _rungs(good, [(["-quality", "80"], {}), (["-quality", "70"], dict(scale=(1, 2)))])
    ok = encoder.recompress_renditions(files, rungs)
    # a 3/8 rung: the single call's code, the message names the rung
    e = _err(lambda: encoder.recompress_renditions(files, [rungs[0], (rungs[1][0], dict(scale=(3, 8)))]))
    assert e.code == A.ERR_UNSUPPORTED and "rendition 1: scale 3/8 gives an IDCT block size of 3" in str(e), str(e)
    e = _err(lambda: encoder.decompress_renditions(files, [{}, dict(scale=(3, 8))]))
    assert e.code == A.ERR_UNSUPPORTED and "rendition 1: " in str(e) and "IDCT block size of 3" in str(e), str(e)
    with pytest.raises(A.B200JpegError):
        encoder.get_output(0)
    # params that do not describe the rung's decoded size
    e = _err(lambda: encoder.recompress_renditions(files, [rungs[0], (rungs[1][0], dict(scale=(1, 4)))]))
    assert e.code == A.ERR_PARAM and "rendition 1: the sources decode to" in str(e), str(e)
    e = _err(lambda: encoder.recompress_renditions(files, [rungs[0], (rungs[0][0], dict(colorspace="gray"))]))
    assert e.code == A.ERR_PARAM and "rendition 1: " in str(e), str(e)
    # an unsupported output colour space and a parameter block that fails validation
    e = _err(lambda: encoder.decompress_renditions(files, [{}, {}, dict(colorspace="rgb565")]))
    assert e.code == A.ERR_UNSUPPORTED and "rendition 2: out_color_space 16" in str(e), str(e)
    bad = rungs[1][0].copy()
    bad.comp_info[0].h_samp_factor = 5                   # MAX_SAMP_FACTOR is 4
    e = _err(lambda: encoder.recompress_renditions(files, [rungs[0], (bad, rungs[1][1])]))
    single = _err(lambda: encoder.recompress(bad, files, **rungs[1][1]))
    assert e.code == single.code and "rendition 1: " in str(e) and _message(single) in str(e), (str(e), str(single))
    # source problems name the image
    truncated = good[:len(good) // 2]
    e = _err(lambda: encoder.recompress_renditions([good, truncated], rungs))
    assert "image 1: " in str(e), str(e)
    from oracle import oracle as OR
    import mozjpeg_b200 as mj
    prog = OR.oracle_encode(mj.params_from_switches(["-progressive"], 200, 136), OR.synth_image(3, 200, 136)).jpeg
    e = _err(lambda: encoder.recompress_renditions([good, prog], rungs))
    assert e.code == A.ERR_UNSUPPORTED and "image 1: progressive" in str(e), str(e)
    e = _err(lambda: encoder.decompress_renditions([good, prog], [kw for _, kw in rungs]))
    assert e.code == A.ERR_UNSUPPORTED and "image 1: progressive" in str(e), str(e)
    with pytest.raises(A.B200JpegError):
        encoder.get_output(0)
    # the encoder recovers; outputs are numbered rung by rung
    assert encoder.recompress_renditions(files, rungs) == ok
    assert encoder.get_output(1 * len(files) + 1) == ok[1][1]
    with pytest.raises(A.B200JpegError, match="no such output"):
        encoder.get_output(len(rungs) * len(files))
    assert encoder.last_scan_bytes() > 0
