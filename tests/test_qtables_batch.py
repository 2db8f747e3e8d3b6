"""Batches with per-image quantization tables (b200jpeg_encode_batch*_qtables, Encoder.encode_batch(..., qtables=)).

Image i of such a batch must be the file the reference writes from a compress object that holds the batch's
parameters with quant_tbl replaced by image i's tables.  The md5s in tests/golden/perimage_q_golden.json were recorded
from the unmodified reference (tools/make_golden.py --perimage-q): per case the base switches, each image's table
switches (-quality, -qtables, -baseline) and the reference's file for base + those switches."""
import hashlib
import json
import os

import numpy as np
import pytest

from common import GOLD

PQ = json.load(open(os.path.join(GOLD, "perimage_q_golden.json")))["cases"]
REFUSED = 73            # the case whose third image holds a table beyond the device trellis divider


def _id(c):
    seed = c["seed"] if isinstance(c["seed"], int) else "%d_12b" % c["seed"][0]
    return "%s:%dx%d:%s%s" % (seed, c["width"], c["height"], "_".join(s.lstrip("-") for s in c["switches"]),
                              ":" + "_".join("%s%d" % (k.split("_")[-1], v) for k, v in c["ext"].items()) if c["ext"] else "")


def _expand(sw):
    return [os.path.join(GOLD, x[6:]) if x.startswith("@GOLD/") else x for x in sw]


def _params(c, i):
    import mozjpeg_b200 as mj
    p = mj.params_from_switches(_expand(c["switches"] + c["images"][i]["switches"]), c["width"], c["height"], 3)
    for k, v in (c["ext"] or {}).items():
        setattr(p, k, v)
    return p


def _image(c, i):
    from mozjpeg_b200.synth import synth_image, synth_image12
    if isinstance(c["seed"], list):
        return synth_image12(c["seed"][0] + i, c["width"], c["height"])
    return synth_image(c["seed"] + i, c["width"], c["height"])


def _batch(c):
    """(parameters of image 0, (N, 4, 64) tables, (N, H, W, 3) images)."""
    ps = [_params(c, i) for i in range(len(c["images"]))]
    qt = np.stack([np.ctypeslib.as_array(p.quant_tbl).copy() for p in ps])
    return ps[0], qt, np.stack([_image(c, i) for i in range(len(c["images"]))])


def _ok(out, rec):
    return len(out) == rec["size"] and hashlib.md5(out).hexdigest() == rec["md5"]


def _seed0(c):
    return c["seed"] if isinstance(c["seed"], int) else c["seed"][0]


# ---------------------------------------------------------------- CPU
@pytest.mark.parametrize("c", PQ, ids=_id)
def test_oracle_matches_recorded_reference(built, c):
    from oracle import oracle as O
    for i, rec in enumerate(c["images"]):
        assert _ok(O.oracle_encode(_params(c, i), _image(c, i)).jpeg, rec), i


@pytest.mark.parametrize("c", PQ, ids=_id)
def test_per_image_parameters_differ_in_tables_only(built, c):
    """The cases are per-image-table batches: apart from quant_tbl (and q_scale_factor, which only feeds the table
    construction) every image's parameter block is image 0's.  cjpeg's -quality >= 80 changing the sampling would
    show up here."""
    import ctypes as C
    from mozjpeg_b200 import _abi as A

    def rest(p):
        q = p.copy()
        for f in ("quant_tbl", "q_scale_factor"):
            C.memset(C.addressof(q) + getattr(A.Params, f).offset, 0, getattr(A.Params, f).size)
        return bytes(q)

    r0 = rest(_params(c, 0))
    for i in range(1, len(c["images"])):
        assert rest(_params(c, i)) == r0, i


@pytest.mark.parametrize("baseline", [False, True])
def test_quality_tables_match_cjpeg_quality(built, baseline):
    import mozjpeg_b200 as mj
    bl = ["-baseline"] if baseline else []
    p0 = mj.params_from_switches(["-sample", "2x2"] + bl, 64, 48, 3)
    got = mj.quality_tables(p0, list(range(1, 101)), force_baseline=baseline)
    for q in range(1, 101):
        want = np.ctypeslib.as_array(mj.params_from_switches(["-quality", str(q), "-sample", "2x2"] + bl, 64, 48, 3).quant_tbl)
        assert np.array_equal(got[q - 1], want), q


def test_transcode_refuses_sources_that_differ_beyond_tables(built):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    im = O.synth_image(5, 64, 48)
    a = O.oracle_encode(mj.params_from_switches(["-quality", "50", "-sample", "2x2"], 64, 48, 3), im).jpeg
    b = O.oracle_encode(mj.params_from_switches(["-quality", "50", "-sample", "1x1"], 64, 48, 3), im).jpeg
    with pytest.raises(ValueError, match="source 1"):
        T.transcode(None, [a, b], [], [])


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("c", PQ, ids=_id)
def test_device_batch_matches_recorded_reference(encoder, c):
    import torch
    import mozjpeg_b200 as mj
    p, qt, imgs = _batch(c)
    if _seed0(c) == REFUSED:
        with pytest.raises(mj.B200JpegError) as ei:
            encoder.encode_batch(p, imgs, qtables=qt)
        assert ei.value.code == mj._abi.ERR_UNSUPPORTED and "image 2" in str(ei.value)
        return
    out = encoder.encode_batch(p, imgs, qtables=qt)
    for i, rec in enumerate(c["images"]):
        assert _ok(out[i], rec), ("host", i)
    t = torch.from_numpy(np.ascontiguousarray(imgs)).cuda()
    encoder.encode_batch_qtables_ptr(p, t.data_ptr(), True, t.stride(1) * t.element_size(), t.stride(0) * t.element_size(), qt)
    torch.cuda.synchronize()
    for i, rec in enumerate(c["images"]):
        assert _ok(encoder.get_output(i), rec), ("device", i)


@pytest.mark.gpu
def test_device_raw_data_per_image_tables(encoder):
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_planes
    from oracle import oracle as O
    w, h = 227, 149
    for sw in (["-baseline", "-sample", "2x2"], ["-fastcrush", "-sample", "2x1"], ["-sample", "2x2"]):
        p = mj.params_from_switches(sw, w, h, 3)
        qs = (30, 90, 60, 75, 45)
        qt = mj.quality_tables(p, qs)
        planes = [synth_planes(p, 80 + i) for i in range(len(qs))]
        stacked = [np.stack([pl[ci] for pl in planes]) for ci in range(p.num_components)]
        got = encoder.encode_batch_raw(p, stacked, qtables=qt)
        for i in range(len(qs)):
            pi = p.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = qt[i]
            assert got[i] == O.oracle_encode_raw(pi, planes[i]), (sw, i)


def _coef_sources(qualities, w=200, h=136, sample="2x2"):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    srcs, planes = [], []
    for i, q in enumerate(qualities):
        r = O.oracle_encode(mj.params_from_switches(["-quality", str(q), "-sample", sample], w, h, 3), O.synth_image(90 + i, w, h), want_debug=True)
        d = r.dbg
        srcs.append(r.jpeg)
        planes.append([np.ascontiguousarray(d["final"][ci][:d["hib"][ci], :d["wib"][ci]]) for ci in range(d["ncomp"])])
    return srcs, planes


@pytest.mark.gpu
def test_device_coefficients_and_transcode_mixed_dqt(encoder):
    """Sources written at different qualities (so with different DQTs): the coefficient entry point with each source's
    tables equals the restatement per source, and transcode() equals the reference's jpegtran per source."""
    from mozjpeg_b200 import jpegtran as T, _abi as A
    from oracle import oracle as O
    srcs, planes = _coef_sources((35, 70, 92, 55, 80))
    stacked = [np.stack([pl[ci] for pl in planes]) for ci in range(len(planes[0]))]
    have_ref = O.ref_available() and os.path.exists(os.path.join(O.REF_DIR, "jpegtran"))
    for tsw in ([], ["-revert"], ["-progressive"], ["-revert", "-optimize"], ["-restart", "1"]):
        got = T.transcode(encoder, srcs, stacked, tsw)
        for i, src in enumerate(srcs):
            p, prefer_smallest = T.params_for_transcode(T.parse_header(src), tsw)
            want = O.oracle_encode_coefs(p, planes[i])
            if prefer_smallest and p.compress_profile == A.PROFILE_MAX_COMPRESSION and len(src) < len(want):
                want = src
            assert got[i] == want, (tsw, i)
            if have_ref:
                assert got[i] == O.ref_jpegtran(src, tsw), (tsw, i)


_INVARIANT = [
    (["-baseline", "-quality", "75", "-sample", "2x2"], 8),
    (["-fastcrush", "-quality", "75", "-sample", "2x2"], 8),
    (["-quality", "75", "-sample", "2x2"], 8),
    (["-precision", "12", "-quality", "75", "-notrellis", "-noovershoot", "-baseline"], 12),
    (["-dct", "float", "-baseline", "-quality", "75"], 8),
    (["-baseline", "-quality", "75", "-smooth", "30"], 8),
    (["-baseline", "-quality", "75", "-restart", "1"], 8),
]


@pytest.mark.gpu
@pytest.mark.parametrize("sw,prec", _INVARIANT, ids=lambda x: "_".join(s.lstrip("-") for s in x) if isinstance(x, list) else str(x))
def test_device_equal_tables_give_encode_batch_files(encoder, sw, prec):
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_image, synth_image12
    w, h, n = 227, 149, 4
    p = mj.params_from_switches(sw, w, h, 3)
    imgs = np.stack([(synth_image12 if prec == 12 else synth_image)(100 + i, w, h) for i in range(n)])
    want = encoder.encode_batch(p, imgs)
    qt = np.repeat(np.ctypeslib.as_array(p.quant_tbl)[None], n, axis=0)
    assert encoder.encode_batch(p, imgs, qtables=qt) == want


@pytest.mark.gpu
def test_device_equal_tables_cmyk_ycck(encoder):
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_image
    w, h, n = 227, 149, 3
    p = mj.tj3_params(w, h, 80, "420", cmyk=True)
    imgs = np.stack([np.concatenate([synth_image(110 + i, w, h), synth_image(120 + i, w, h)[..., :1]], axis=2) for i in range(n)])
    want = encoder.encode_batch(p, imgs)
    qt = np.repeat(np.ctypeslib.as_array(p.quant_tbl)[None], n, axis=0)
    got = encoder.encode_batch(p, imgs, qtables=qt)
    assert got == want
    # and per-image tables against the restatement of the CMYK->YCCK conversion
    import colorspace_cases as CC
    qt = mj.quality_tables(p, (30, 75, 95))
    got = encoder.encode_batch(p, imgs, qtables=qt)
    for i in range(n):
        pi = p.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = qt[i]
        assert got[i] == CC.oracle_encode(pi, imgs[i]).jpeg, i


@pytest.mark.gpu
def test_device_kernel_launches_equal_encode_batch(encoder):
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_image
    w, h = 227, 149
    for sw in (["-baseline", "-sample", "2x2"], ["-sample", "2x2"], ["-fastcrush", "-sample", "2x2"]):
        p = mj.params_from_switches(sw, w, h, 3)
        imgs = np.stack([synth_image(130 + i, w, h) for i in range(6)])
        qt = mj.quality_tables(p, (20, 50, 75, 90, 95, 60))
        a = encoder.kernel_launches(); encoder.encode_batch(p, imgs)
        b = encoder.kernel_launches(); encoder.encode_batch(p, imgs, qtables=qt)
        c = encoder.kernel_launches()
        assert c - b == b - a, sw


def _single(encoder, p, img, q):
    pi = p.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = q
    return encoder.encode_batch(pi, img[None])[0]


@pytest.mark.gpu
@pytest.mark.parametrize("sw", [["-baseline", "-sample", "2x2"], ["-sample", "2x2"], ["-fastcrush", "-sample", "2x1", "-dct", "float"]],
                         ids=lambda x: "_".join(s.lstrip("-") for s in x))
def test_device_ladder_zero_stride(encoder, sw):
    """One image at 8 qualities, input shared by every image (stride 0), from host and from device memory.  1024 RGB
    pixels make a 3072-byte row pitch, so the forward kernel loads its interior tiles by TMA from one tensor map that
    every image addresses as image 0."""
    import torch
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_image
    w, h = 1024, 576
    p = mj.params_from_switches(sw, w, h, 3)
    img = synth_image(140, w, h)
    qt = mj.quality_tables(p, (40, 50, 60, 70, 80, 85, 90, 95))
    want = [_single(encoder, p, img, q) for q in qt]
    assert encoder.encode_batch(p, img[None], qtables=qt) == want
    t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    encoder.encode_batch_qtables_ptr(p, t.data_ptr(), True, t.stride(0), 0, qt)
    torch.cuda.synchronize()
    assert [encoder.get_output(i) for i in range(len(qt))] == want


@pytest.mark.gpu
@pytest.mark.parametrize("streams", [1, 2])
def test_device_table_sets_across_chunks(encoder, streams):
    """Sets that change inside and across chunk boundaries (3 images per chunk, a ragged last chunk of 2).  The 227-pixel
    width loads pixels per thread; at 1024 pixels (a 16-byte-aligned row pitch) the TMA path reads the per-image sets."""
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_image
    n = 11
    for w, h in ((227, 149), (1024, 136)):
        for sw in (["-baseline", "-sample", "2x2"], ["-sample", "2x2"]):
            p = mj.params_from_switches(sw, w, h, 3)
            ladder = mj.quality_tables(p, (30, 60, 90, 75))
            qt = ladder[[0, 0, 1, 1, 2, 3, 3, 0, 2, 1, 1]]
            imgs = np.stack([synth_image(150 + i, w, h) for i in range(n)])
            want = [_single(encoder, p, imgs[i], qt[i]) for i in range(n)]
            encoder.set_chunk_images(3); encoder.set_streams(streams)
            try:
                got = encoder.encode_batch(p, imgs, qtables=qt)
                assert encoder.chunk_images() == 3
            finally:
                encoder.set_chunk_images(0); encoder.set_streams(2)
            assert got == want, (w, sw)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [0, 32768, 65535])
def test_device_out_of_range_entry_is_param_error(encoder, bad):
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_image
    w, h = 64, 48
    p = mj.params_from_switches(["-baseline", "-sample", "2x2"], w, h, 3)
    qt = mj.quality_tables(p, (50, 75, 90))
    qt[1, 1, 17] = bad
    with pytest.raises(mj.B200JpegError) as ei:
        encoder.encode_batch(p, np.stack([synth_image(160 + i, w, h) for i in range(3)]), qtables=qt)
    assert ei.value.code == mj._abi.ERR_PARAM and "image 1" in str(ei.value) and "table 1" in str(ei.value)


@pytest.mark.gpu
def test_device_raw_and_coefficients_zero_stride(encoder):
    """One image's planes (raw data) or blocks (coefficients) shared by every image of the batch: host input staged once,
    each file as if encoded alone with its tables."""
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_planes
    from oracle import oracle as O
    w, h = 227, 149
    p = mj.params_from_switches(["-baseline", "-sample", "2x2"], w, h, 3)
    qt = mj.quality_tables(p, (25, 50, 75, 90, 97))
    planes = synth_planes(p, 170)
    encoder.set_chunk_images(2)                        # three chunks read the one staged copy
    try:
        got = encoder.encode_batch_raw(p, [a[None] for a in planes], qtables=qt)
    finally:
        encoder.set_chunk_images(0)
    for i in range(len(qt)):
        pi = p.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = qt[i]
        assert got[i] == O.oracle_encode_raw(pi, planes), ("raw", i)
    srcs, coefs = _coef_sources((60,), w=w, h=h)
    pc = p.copy(); pc.trellis_quant = 0
    got = encoder.encode_batch_coefs(pc, [a[None] for a in coefs[0]], qtables=qt)
    for i in range(len(qt)):
        pi = pc.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = qt[i]
        assert got[i] == O.oracle_encode_coefs(pi, coefs[0]), ("coefs", i)


@pytest.mark.parametrize("bad", [65537, -1, 1.5])
def test_qtables_that_do_not_fit_uint16_are_refused(built, bad):
    """65537 would wrap to 1 and pass the library's range check: the binding refuses it before converting."""
    import mozjpeg_b200 as mj
    qt = np.full((2, 4, 64), 16, dtype=np.float64 if isinstance(bad, float) else np.int64)
    qt[1, 0, 5] = bad
    with pytest.raises(ValueError, match="0..65535"):
        mj.Encoder._qtables(qt, 2)
