"""YUV encoding (tj3EncodeYUVPlanes8 / tj3EncodeYUV8) on the device: plane geometry and refusals on the CPU, the planes
byte for byte against the reference's (tests/golden/yuv_golden.json) on the GPU, and the TurboJPEG interposer under the
reference's tjbench and a small C application."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from common import GOLD, ROOT
import yuv_cases as Y

SHIM = os.path.join(ROOT, "integration", "_build", "libjpeg_b200shim.so")
TJBENCH = os.path.join(ROOT, "oracle", "_ref", "tjbench")
need_ref = pytest.mark.skipif(not os.path.exists(Y.REF_TJ), reason="oracle/_ref/libturbojpeg_ref.so not built (needs the reference at build time)")


def golden():
    with open(os.path.join(GOLD, "yuv_golden.json")) as f:
        return json.load(f)["cases"]


def params(pf, subsamp, w, h):
    """setCompDefaults for tj3EncodeYUVPlanes8: unlike tj3Compress8 it does not turn TJPF_GRAY into TJSAMP_GRAY, so the
    default colour space follows the subsampling alone."""
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    cs = A.CS_GRAYSCALE if subsamp == "gray" else A.CS_YCCK if pf == "CMYK" else A.CS_YCbCr
    return mj.tj3_params(w, h, subsamp=subsamp, pixel_format=pf, colorspace=cs)


def dims(size):
    return (227, 149) if size == "testorig" else tuple(int(v) for v in size.split("x"))


# ---------------------------------------------------------------------------- CPU
@need_ref
def test_plane_dims_equal_tj3YUVPlaneWidth_and_Height(built):
    import mozjpeg_b200 as mj
    ref = Y.RefTJ()
    try:
        for ss in Y.SUBSAMPS:
            for w in (1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 31, 33, 227, 1920, 3841):
                for h in (1, 2, 3, 5, 8, 13, 149, 1080, 2161):
                    p = params("RGB", ss, w, h)
                    for ci in range(p.num_components):
                        assert mj.yuv_plane_dims(p, ci) == ref.plane_dims(ci, w, h, ss), (ss, w, h, ci)
    finally:
        ref.close()


def test_golden_refusals_are_the_c_abi_refusals(built):
    """Every colour pair the reference refuses, b200jpeg_validate refuses too; every case it codes validates.  CMYK pixels
    are refused by TurboJPEG before a parameter block exists (the interposer hands them over; the entry point refuses
    4-component blocks, checked on the GPU)."""
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    lib = A.load()
    seen = set()
    for c in golden():
        key = (c["pf"], c["subsamp"])
        if key in seen:
            continue
        seen.add(key)
        if c["pf"] == "CMYK":
            assert "CMYK" in c["error"]
            continue
        p = params(c["pf"], c["subsamp"], 33, 19)
        rc = lib.b200jpeg_validate(p)
        assert (rc != 0) == ("error" in c), (key, rc, c.get("error"))
    assert len(seen) == 7 * 12


def test_golden_covers_the_matrix():
    cases = golden()
    assert len(cases) == len(Y.SUBSAMPS) * len(Y.PIXEL_FORMATS) * len(Y.SIZES) * len(Y.PADS)
    assert sum("error" not in c for c in cases) > 900


# ---------------------------------------------------------------------------- GPU
def _torch_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
def test_every_golden_case_on_the_device(encoder):
    """Host in / host out for NULL strides; padded plane pitch with sentinels for the others."""
    from mozjpeg_b200 import _abi as A
    import mozjpeg_b200 as mj
    pix_cache = {}
    for c in golden():
        key = (c["size"], c["pf"])
        if key not in pix_cache:
            pix_cache = {key: Y.case_pixels("testorig" if c["size"] == "testorig" else dims(c["size"]), c["pf"])}
        pix = pix_cache[key]
        h, w = pix.shape[:2]
        p = params(c["pf"], c["subsamp"], w, h)
        if "error" in c:
            with pytest.raises(A.B200JpegError) as ei:
                encoder.encode_yuv_batch(p, pix[None])
            # CMYK: the 4-component YCCK block is beyond the device path, the grayscale one an invalid colour pair
            assert ei.value.code in ((A.ERR_UNSUPPORTED, A.ERR_PARAM) if c["pf"] == "CMYK" else (A.ERR_PARAM,)), c
            continue
        if c["pad"] == 0:
            planes = encoder.encode_yuv_batch(p, pix[None])[0]
        else:
            bufs = [np.full((ph, pw + c["pad"]), 0xEE, np.uint8) for pw, ph in c["dims"]]
            encoder.encode_yuv_batch_ptr(p, pix.ctypes.data, False, pix.strides[0], pix.size, [b.ctypes.data for b in bufs], False,
                                         [b.strides[0] for b in bufs], [b.size for b in bufs], 1)
            for b, (pw, _) in zip(bufs, c["dims"]):
                assert (b[:, pw:] == 0xEE).all(), ("pitch padding written", c)
            planes = [b[:, :pw] for b, (pw, _) in zip(bufs, c["dims"])]
        assert [list(q.shape[::-1]) for q in planes] == c["dims"], c
        assert [Y.md5(q) for q in planes] == c["md5"], c


BATCH_CASES = [("RGB", "420", (33, 19)), ("BGRX", "411", (1920, 1080)), ("XRGB", "441", (17, 1)), ("GRAY", "gray", "testorig"),
               ("ABGR", "440", (7, 5)), ("BGR", "422", "testorig"), ("RGBA", "444", (1, 17))]


@pytest.mark.gpu
@pytest.mark.parametrize("pf,ss,size", BATCH_CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("where", ["host-host", "dev-host", "host-dev", "dev-dev"])
def test_batch_of_five_with_padded_strides(encoder, pf, ss, size, where):
    """Five images with a padded image stride and plane pitch and a gap between images, input and output in host or
    device memory; sentinel bytes in the pitch padding and between the images stay as they were."""
    import torch
    from mozjpeg_b200 import yuv_plane_dims
    imgs = [Y.case_pixels(size, pf) if i == 0 else Y.to_pixel_format(Y.synth_rgb(100 + i, *Y.case_pixels(size, pf).shape[1::-1]), pf, i)
            for i in range(5)]
    h, w, ps = imgs[0].shape
    row_pitch, image_stride = w * ps + 7, (w * ps + 7) * h + 29
    src = np.zeros(image_stride * 5, np.uint8)
    for i, im in enumerate(imgs):
        for y in range(h):
            src[i * image_stride + y * row_pitch: i * image_stride + y * row_pitch + w * ps] = im[y].reshape(-1)
    p = params(pf, ss, w, h)
    ref = Y.RefTJ()
    want = [ref.encode_planes(im, pf, ss)[0] for im in imgs]
    ref.close()
    geo = [yuv_plane_dims(p, ci) for ci in range(p.num_components)]
    pitch = [pw + 11 + ci for ci, (pw, _) in enumerate(geo)]
    stride = [pt * ph + 37 for pt, (_, ph) in zip(pitch, geo)]
    outs = [np.full(st * 5, 0xEE, np.uint8) for st in stride]
    src_on_dev, dst_on_dev = where.startswith("dev"), where.endswith("dev")
    s_t = _torch_dev(src) if src_on_dev else None
    o_t = [_torch_dev(o) for o in outs] if dst_on_dev else None
    torch.cuda.synchronize()               # the encoder's stream does not wait for torch's
    encoder.encode_yuv_batch_ptr(p, s_t.data_ptr() if src_on_dev else src.ctypes.data, src_on_dev, row_pitch, image_stride,
                                 [t.data_ptr() for t in o_t] if dst_on_dev else [o.ctypes.data for o in outs], dst_on_dev, pitch, stride, 5)
    if dst_on_dev:
        torch.cuda.synchronize()
        outs = [t.cpu().numpy() for t in o_t]
    for ci, ((pw, ph), pt, st, o) in enumerate(zip(geo, pitch, stride, outs)):
        for i in range(5):
            block = o[i * st: i * st + pt * ph].reshape(ph, pt)
            assert np.array_equal(block[:, :pw], want[i][ci]), (where, i, ci)
            assert (block[:, pw:] == 0xEE).all(), ("pitch padding written", where, i, ci)
            assert (o[i * st + pt * ph: (i + 1) * st] == 0xEE).all(), ("gap between images written", where, i, ci)
    st = encoder.stage_times()
    assert "encode_yuv" in st
    if not src_on_dev:
        assert "h2d" in st
    if not dst_on_dev:
        assert "d2h" in st


@pytest.mark.gpu
def test_refusals(encoder):
    from mozjpeg_b200 import _abi as A
    import mozjpeg_b200 as mj
    img = Y.case_pixels((33, 19), "RGB")[None]

    def code(p, **kw):
        with pytest.raises(A.B200JpegError) as ei:
            if kw:
                encoder.encode_yuv_batch_ptr(p, img.ctypes.data, False, 33 * 3, img.size, kw["planes"], False, kw["pitch"], kw["stride"], kw.get("n", 1))
            else:
                encoder.encode_yuv_batch(p, img)
        return ei.value.code

    p = params("RGB", "420", 33, 19)
    q = p.copy(); A.check(A.load().b200jpeg_enable_lossless(q, 1, 0), "enable_lossless"); q.trellis_quant = 0
    assert code(q) == A.ERR_PARAM
    q = p.copy(); q.smoothing_factor = 10
    assert code(q) == A.ERR_UNSUPPORTED
    q = p.copy(); q.comp_info[1].h_samp_factor = 2
    assert code(q) == A.ERR_UNSUPPORTED
    buf = np.zeros(1 << 16, np.uint8)
    ptrs = [buf.ctypes.data] * 3
    assert code(p, planes=ptrs, pitch=[33, 17, 17], stride=[0, 0, 0]) == A.ERR_PARAM          # pw0 = 34
    assert code(p, planes=ptrs, pitch=[34, 17, 17], stride=[34 * 20 - 1, 17 * 10, 17 * 10], n=2) == A.ERR_PARAM


@need_ref
@pytest.mark.gpu
@pytest.mark.skipif(not (os.path.exists(SHIM) and os.path.exists(TJBENCH)), reason="shim / reference tjbench not built")
@pytest.mark.parametrize("opts", [["-subsamp", "420"], ["-subsamp", "422", "-optimize"], ["-subsamp", "444"], ["-subsamp", "gray"]],
                         ids=lambda s: "_".join(x.lstrip("-") for x in s))
@pytest.mark.parametrize("fmt", [None, "-rgb", "-rgbx", "-bgrx", "-xbgr", "-xrgb"], ids=lambda f: (f or "-bgr").lstrip("-"))
def test_tjbench_yuv_runs_on_the_device(opts, fmt, tmp_path):
    """tjbench -yuv: tj3EncodeYUV8 (colour conversion + downsampling) and then tj3CompressFromYUVPlanes8 ->
    jpeg_write_raw_data, both on the device; the files equal the reference's own."""
    outs = []
    for name, env_extra in (("dev", {"LD_PRELOAD": SHIM, "B200_SHIM_REQUIRE": "1", "B200_SHIM_VERBOSE": "1"}), ("ref", {})):
        d = tmp_path / name
        d.mkdir()
        shutil.copyfile(os.path.join(GOLD, "testorig.ppm"), d / "img.ppm")
        r = subprocess.run([TJBENCH, "img.ppm", "75", *([fmt] if fmt else []), "-quiet", "-benchtime", "0.01", "-warmup", "0", "-componly", "-yuv", *opts],
                           cwd=d, env=dict(os.environ, **env_extra), capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr + r.stdout
        if name == "dev":
            assert "device path (YUV planes" in r.stderr, r.stderr
            assert "reference path" not in r.stderr, r.stderr
        jpgs = sorted(f for f in os.listdir(d) if f.endswith(".jpg"))
        assert len(jpgs) == 1, os.listdir(d)
        outs.append((d / jpgs[0]).read_bytes())
    assert outs[0] == outs[1] and len(outs[0]) > 100


@need_ref
@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(SHIM), reason="shim not built")
def test_c_application_under_the_interposer(tmp_path):
    """tests/refyuv.c: tj3EncodeYUV8 at alignments 1, 4, 64 and tj3EncodeYUVPlanes8 with explicit strides write the
    same whole buffers (padding included) with the interposer preloaded as without it."""
    import hashlib
    ref = os.path.join(ROOT, "oracle", "_ref")
    exe = tmp_path / "refyuv"
    subprocess.check_call(["gcc", "-O2", "-w", "-I" + os.path.join(ref, "inc"), "-o", str(exe), os.path.join(ROOT, "tests", "refyuv.c"),
                           "-L" + ref, "-lturbojpeg_ref", "-Wl,-rpath," + ref])
    sums = []
    for name, env_extra in (("dev", {"LD_PRELOAD": SHIM, "B200_SHIM_REQUIRE": "1", "B200_SHIM_VERBOSE": "1"}), ("ref", {})):
        d = tmp_path / name
        d.mkdir()
        r = subprocess.run([str(exe), str(d)], env=dict(os.environ, **env_extra), capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        if name == "dev":
            assert r.stderr.count("device path (YUV planes") == (7 * 3 + 1) * 4, r.stderr
        sums.append({f: hashlib.md5((d / f).read_bytes()).hexdigest() for f in sorted(os.listdir(d))})
    assert len(sums[0]) == 22 * 3 + 18 * 3 + 4 and sums[0] == sums[1]      # 22 (subsampling, format) pairs, 18 of them with chroma
