"""Decompression to YUV planes (b200jpeg_decompress_yuv_batch, tj3DecompressToYUVPlanes8): plane sizes and
subsampling on the CPU, and on the GPU every case of tests/yuv_decode_cases.py against the reference's planes recorded
in tests/golden/yuv_decode_golden.json (the samples the reference leaves to its heap masked out)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import yuv_decode_cases as Y
import mozjpeg_b200 as mj
from mozjpeg_b200 import _abi as A

GOLD = {c["id"]: c for c in Y.golden()["cases"]}
CASES = Y.cases()
DEVICE_SCALES = {(1, 8), (1, 4), (1, 2), (1, 1)}


def _info(src):
    info = A.SourceInfo()
    A.check(mj._lib.b200jpeg_parse_source(src, len(src), C.byref(info)), "parse_source")
    return info


def _code(fn, *a, **kw):
    try:
        fn(*a, **kw)
    except mj.B200JpegError as e:
        return e.code, str(e)
    return 0, ""


# ------------------------------------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize("cid", [c[0] for c in CASES if "error" not in GOLD[c[0]] and c[2] in DEVICE_SCALES])
def test_dims_match_the_reference(cid):
    """decompress_yuv_dims gives the reference's TJSAMP_* and plane sizes, and the restatement in yuv_decode_cases."""
    _, sid, scale, dct = next(c for c in CASES if c[0] == cid)
    g = GOLD[cid]
    info = _info(Y.source(sid))
    ss, dims = mj.decompress_yuv_dims(info, scale=scale, dct=dct)
    assert ss == g["subsamp"] and [list(d) for d in dims] == g["dims"]
    rss, rdims = Y.plan(info, scale)
    assert Y.SUBSAMPS[rss] == ss and [d[:2] for d in rdims] == [tuple(d) for d in dims]


def test_subsampling_of_every_factor_combination():
    """getSubsamp as the library states it, for every 3-component factor combination 1..4 and gray, against the Python
    restatement; TJSAMP_UNKNOWN is the reference's refusal."""
    info = A.SourceInfo()
    info.image_width, info.image_height, info.num_components, info.jpeg_color_space = 64, 48, 3, A.CS_YCbCr
    fs = [(h, v) for h in range(1, 5) for v in range(1, 5)]
    seen = set()
    for f0 in fs:
        for f1 in fs:
            for f2 in (f1, (1, 1)):
                for c, (h, v) in enumerate((f0, f1, f2)):
                    info.h_samp_factor[c], info.v_samp_factor[c] = h, v
                want = Y.tj_subsamp(info)
                code, msg = _code(mj.decompress_yuv_dims, info)
                if want < 0:
                    assert code == A.ERR_PARAM and "Could not determine subsampling level of JPEG image" in msg
                else:
                    assert code == 0 and mj.decompress_yuv_dims(info)[0] == Y.SUBSAMPS[want]
                    seen.add(want)
    assert seen == {0, 1, 2, 4, 5, 6}
    info.num_components, info.jpeg_color_space = 1, A.CS_GRAYSCALE
    assert mj.decompress_yuv_dims(info)[0] == "gray"


def test_option_validation():
    info = _info(Y.source("y_420"))
    for kw in ({"dct": "float"}, {"fancy": False}, {"colorspace": "rgb"}, {"scale": (1, 3)}, {"scale": (2, 4)}):
        code, msg = _code(mj.decompress_yuv_dims, info, **kw)
        assert code == A.ERR_PARAM, (kw, msg)
    for sc in Y.REFUSED_SCALES + [(2, 1), (7, 8)]:
        code, msg = _code(mj.decompress_yuv_dims, info, scale=sc)
        assert code == A.ERR_UNSUPPORTED and "IDCT block size of %d" % (8 * sc[0] // sc[1]) in msg
    o = mj.decompress_options()
    w = C.c_int()
    assert mj._lib.b200jpeg_decompress_yuv_dims(C.byref(info), C.byref(o), 3, C.byref(w), None, None) == A.ERR_PARAM
    code, msg = _code(mj.decompress_yuv_dims, _info(Y.source("prog:cmyk")))
    assert code == A.ERR_PARAM and "JPEG image must have 3 or fewer components" in msg


@pytest.mark.skipif(not os.path.exists(Y.REF_TJ), reason="reference TurboJPEG library not built")
def test_packed_layout_matches_tj3YUVBufSize():
    ref = Y.RefTJ()
    try:
        for w, h in ((1, 1), (7, 5), (227, 149), (1920, 1080)):
            for ss in range(7):
                dims = [Y.plane_dims(ci, w, h, ss) for ci in range(1 if ss == 3 else 3)]
                for align in (1, 2, 4, 32, 64):
                    offs, pitches, total = mj.yuv_packed_layout(dims, align)
                    assert total == ref.buf_size(w, align, h, ss)
                    assert offs[0] == 0 and all(offs[i + 1] == offs[i] + pitches[i] * dims[i][1] for i in range(len(dims) - 1))
                    assert all(p % align == 0 and p >= d[0] for p, d in zip(pitches, dims))
    finally:
        ref.close()
    with pytest.raises(ValueError):
        mj.yuv_packed_layout([(3, 3)], 3)


# ------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope="module")
def enc():
    e = mj.Encoder(0)
    yield e
    e.close()


def _opts(scale, dct):
    return {"scale": scale, "dct": dct}


def _check_planes(got, g, info, scale):
    _, dims = Y.plan(info, scale)
    assert [list(p.shape[::-1]) for p in got] == g["dims"]
    assert [Y.md5(Y.defined(p, *d)) for p, d in zip(got, dims)] == g["md5"]


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c[0] for c in CASES])
def test_matches_the_reference(enc, cid):
    """Every case: the reference's planes (defined samples), or the device's refusal of what it refuses."""
    _, sid, scale, dct = next(c for c in CASES if c[0] == cid)
    g = GOLD[cid]
    src = Y.source(sid)
    enc.set_progressive_decode(sid.startswith("prog:"))
    try:
        if scale not in DEVICE_SCALES:
            code, msg = _code(enc.decompress_yuv, [src], **_opts(scale, dct))
            assert code == A.ERR_UNSUPPORTED and "IDCT block size" in msg
        elif sid == "prog:drop_to_dc_only":
            code, msg = _code(enc.decompress_yuv, [src], **_opts(scale, dct))
            assert code == A.ERR_UNSUPPORTED and "block smoothing" in msg and "image 0:" in msg
        elif sid == "prog:corrupt":
            code, msg = _code(enc.decompress_yuv, [src], **_opts(scale, dct))
            assert code == A.ERR_BAD_SOURCE and "image 0:" in msg
        elif "error" in g:
            code, msg = _code(enc.decompress_yuv, [src], **_opts(scale, dct))
            assert code == A.ERR_PARAM and "image 0: " + g["error"].split("(): ")[-1] in msg, (msg, g["error"])
        else:
            got = enc.decompress_yuv([src], **_opts(scale, dct))[0]
            _check_planes(got, g, _info(src), scale)
            st = enc.stage_times()
            assert "idct" in st and "upsample_color" not in st
    finally:
        enc.set_progressive_decode(False)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", ["y_411:1/4:int", "y_420:1/8:int", "y_2x3:1/2:int", "y_ns422:1/2:fast", "y_gray:1/1:fast"])
def test_prefilled_bytes_stay(enc, cid):
    """Host and device destinations with padded rows and gaps between images, prefilled with 0xEE: the defined samples
    match the reference, every other byte (pitch padding, gaps, the masked columns and rows) is still 0xEE, and both
    destinations hold the same bytes."""
    import torch
    _, sid, scale, dct = next(c for c in CASES if c[0] == cid)
    g = GOLD[cid]
    src = Y.source(sid)
    info = _info(src)
    _, dims = Y.plan(info, scale)
    n = 3
    pitch = [d[0] + 5 for d in dims]
    stride = [p * d[1] + 7 for p, d in zip(pitch, dims)]
    host = [np.full(s * n, 0xEE, np.uint8) for s in stride]
    ptrs = [h.ctypes.data for h in host]
    o = mj.decompress_options(**_opts(scale, dct))
    bufs, fp, sizes = enc._files([src] * n)
    k = len(dims)
    A.check(mj._lib.b200jpeg_decompress_yuv_batch(enc._h, C.byref(o), fp, sizes, n, (C.c_void_p * k)(*ptrs), 0, (C.c_size_t * k)(*pitch),
                                                   (C.c_size_t * k)(*stride)), "decompress_yuv_batch")
    dev = [torch.full((s * n,), 0xEE, dtype=torch.uint8, device="cuda") for s in stride]
    enc.decompress_yuv_ptr([src] * n, [t.data_ptr() for t in dev], pitch, stride, **_opts(scale, dct))
    torch.cuda.synchronize()
    for c, (pw, ph, iw, ih) in enumerate(dims):
        assert np.array_equal(host[c], dev[c].cpu().numpy())
        mask = np.zeros(stride[c] * n, bool)
        for i in range(n):
            for y in range(min(ih, ph)):
                mask[i * stride[c] + y * pitch[c]:i * stride[c] + y * pitch[c] + min(iw, pw)] = True
        assert (host[c][~mask] == 0xEE).all()
        for i in range(n):
            plane = np.lib.stride_tricks.as_strided(host[c][i * stride[c]:], (ph, pw), (pitch[c], 1))
            assert Y.md5(Y.defined(plane, pw, ph, iw, ih)) == g["md5"][c]


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 2])
def test_batch_of_mixed_tables_equals_single_calls(enc, chunk):
    """One batch of 200x136 4:2:0 sources with different tables, restarts and scan layouts equals the single-image
    calls, whole or in chunks of two images."""
    sids = ["q5", "q100", "sof1_dqt16", "restart_1", "multi_scan"]
    srcs = [Y.source(s) for s in sids]
    for dct, scale in (("int", (1, 1)), ("fast", (1, 2)), ("int", (1, 4))):
        singles = [enc.decompress_yuv([s], scale=scale, dct=dct)[0] for s in srcs]
        enc.set_chunk_images(chunk)
        try:
            batch = enc.decompress_yuv(srcs, scale=scale, dct=dct)
            if chunk:
                assert enc.chunk_images() == chunk
        finally:
            enc.set_chunk_images(0)
        for a, b in zip(singles, batch):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_refusals_name_the_image_and_leave_the_encoder_usable(enc):
    """Refused batches name the image, launch no kernel (the refusal comes before any device work) and leave the
    encoder usable."""
    good = Y.source("y_420")
    for bad, code in (("prog:cmyk", A.ERR_PARAM), ("prog:sample_3x2", A.ERR_PARAM), ("prog:prog12", A.ERR_PARAM), ("y_444", A.ERR_PARAM),
                      ("prog:drop_to_dc_only", A.ERR_UNSUPPORTED)):
        enc.set_progressive_decode(True)
        try:
            before = enc.kernel_launches()
            c, msg = _code(enc.decompress_yuv, [good, good, Y.source(bad)])
            assert enc.kernel_launches() == before, bad
        finally:
            enc.set_progressive_decode(False)
        assert c == code and re.search(r"image 2: ", msg), (bad, msg)
    before = enc.kernel_launches()
    c, msg = _code(enc.decompress_yuv, [Y.source("prog:progressive")])
    assert c == A.ERR_UNSUPPORTED and "image 0:" in msg and enc.kernel_launches() == before
    got = enc.decompress_yuv([good])[0]
    _check_planes(got, GOLD["y_420:1/1:int"], _info(good), (1, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("sid,scale,dct", Y.RECOMPRESS, ids=[Y.case_id(*c) for c in Y.RECOMPRESS])
def test_planes_recompress_as_the_reference(enc, sid, scale, dct):
    """decompress_yuv then encode_batch_raw(tj3_params(.., 75, subsampling)) is the reference's
    tj3DecompressToYUVPlanes8 then tj3CompressFromYUVPlanes8, byte for byte.  tj3CompressFromYUVPlanes8 extends each
    plane to whole blocks by repeating its last column and row; the raw-data entry point takes the extended planes."""
    g = {c["id"]: c for c in Y.golden()["recompress"]}[Y.case_id(sid, scale, dct)]
    src = Y.source(sid)
    info = _info(src)
    ss, dims = mj.decompress_yuv_dims(info, scale=scale, dct=dct)
    planes = enc.decompress_yuv([src], scale=scale, dct=dct)[0]
    k = 8 * scale[0] // scale[1]
    ow, oh = -(-info.image_width * k // 8), -(-info.image_height * k // 8)
    p = mj.tj3_params(ow, oh, quality=75, subsamp=ss)
    hmax = max(p.comp_info[c].h_samp_factor for c in range(p.num_components))
    vmax = max(p.comp_info[c].v_samp_factor for c in range(p.num_components))
    ext = []
    for c, a in enumerate(planes):
        wib = -(-ow * p.comp_info[c].h_samp_factor // (hmax * 8)); hib = -(-oh * p.comp_info[c].v_samp_factor // (vmax * 8))
        ext.append(np.pad(a, ((0, hib * 8 - a.shape[0]), (0, wib * 8 - a.shape[1])), mode="edge")[None])
    out = enc.encode_batch_raw(p, ext)[0]
    assert len(out) == g["size"] and Y.md5(np.frombuffer(out, np.uint8)) == g["md5"]


DEC_GOLD = {c["id"]: c for c in Y.golden()["decode"]}


def _decode_params(ss, w, h, pf):
    cs = A.CS_GRAYSCALE if ss == "gray" else A.CS_YCbCr
    return mj.tj3_params(w, h, subsamp=ss, pixel_format=pf, colorspace=cs)


@pytest.mark.gpu
@pytest.mark.parametrize("did", [c[0] for c in Y.decode_cases()])
def test_decode_matches_the_reference(enc, did):
    """tj3DecodeYUVPlanes8 on seeded planes, every subsampling x pixel format x size x plane pitch: the reference's
    pixels, or its refusal of CMYK before any device work."""
    _, ss, (w, h), pf, pad = next(c for c in Y.decode_cases() if c[0] == did)
    g = DEC_GOLD[did]
    p = _decode_params(ss, w, h, pf)
    planes = Y.decode_planes(ss, w, h)
    if "error" in g:
        before = enc.kernel_launches()
        code, msg = _code(enc.decode_yuv, p, [planes])
        assert code == A.ERR_PARAM and g["error"].split("(): ")[-1] in msg and enc.kernel_launches() == before
        return
    if pad == 0:
        out = enc.decode_yuv(p, [planes])[0]
    else:                                      # pitched host planes, the padding filled with bytes that must not be read
        bufs = [np.full((a.shape[0], a.shape[1] + pad), 0xEE, np.uint8) for a in planes]
        for b, a in zip(bufs, planes):
            b[:, :a.shape[1]] = a
        out = np.full((h, w, g["shape"][2]), 0x11, np.uint8)
        enc.decode_yuv_ptr(p, [b.ctypes.data for b in bufs], False, [b.strides[0] for b in bufs], [b.nbytes for b in bufs],
                           out.ctypes.data, False, out.strides[0], out.nbytes, 1)
    assert list(out.shape) == g["shape"] and Y.md5(out) == g["md5"]
    assert "yuv_to_pixels" in enc.stage_times()


@pytest.mark.gpu
@pytest.mark.parametrize("ss", Y.SUBSAMPS)
def test_decode_device_batch_equals_host_single_calls(enc, ss):
    """A batch of three images with planes and pixels in device memory (pitched, gaps between images, prefilled with
    0xEE) equals the single host calls, and leaves every byte outside the pixel rows as it was."""
    import torch
    w, h, n = 227, 149, 3
    p = _decode_params(ss, w, h, "BGRX")
    singles = []
    per = []
    for i in range(n):
        planes = [np.roll(a, 7 * i, axis=1) for a in Y.decode_planes(ss, w, h)]
        per.append(planes)
        singles.append(enc.decode_yuv(p, [planes])[0])
    pitch = [a.shape[1] + 3 for a in per[0]]
    stride = [pt * a.shape[0] + 5 for pt, a in zip(pitch, per[0])]
    dev_planes = []
    for c, a0 in enumerate(per[0]):
        buf = np.full(stride[c] * n, 0xEE, np.uint8)
        for i in range(n):
            v = np.lib.stride_tricks.as_strided(buf[i * stride[c]:], a0.shape, (pitch[c], 1))
            v[:] = per[i][c]
        dev_planes.append(torch.from_numpy(buf).cuda())
    rp, st = w * 4 + 8, (w * 4 + 8) * h + 16
    pix = torch.full((st * n,), 0xEE, dtype=torch.uint8, device="cuda")
    enc.decode_yuv_ptr(p, [t.data_ptr() for t in dev_planes], True, pitch, stride, pix.data_ptr(), True, rp, st, n)
    got = pix.cpu().numpy()
    mask = np.zeros(st * n, bool)
    for i in range(n):
        img = np.lib.stride_tricks.as_strided(got[i * st:], (h, w * 4), (rp, 1))
        assert np.array_equal(img.reshape(h, w, 4), singles[i])
        for y in range(h):
            mask[i * st + y * rp:i * st + y * rp + w * 4] = True
    assert (got[~mask] == 0xEE).all()
