"""Decompressing at every scale the reference takes (all_scales): jidctint.c's scaled IDCTs of block sizes 3, 5, 6, 7
and 9 .. 16 on the device, through every route that decodes to pixels or planes, against what the reference makes
with the same options (tests/golden/idct_scaling_golden.json, recorded by tools/make_golden.py --idct-scaling;
tests/refdecopt.c where the reference build exists).  On the CPU: the golden's coverage, the size queries, the numpy
restatement of the IDCTs against every gray case, the generated device functions, and the refusal without the flag."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import common  # noqa: F401,E402  (puts the repository root on sys.path)
import decompress_options_cases as O  # noqa: E402
import idct_scaling_cases as S  # noqa: E402
import yuv_decode_cases as Y  # noqa: E402

GOLD = S.golden()
CASES = {c[0]: c for c in S.cases()}
PIX = {c["id"]: c for c in GOLD["cases"]}
YUV = {c["id"]: c for c in GOLD["yuv"]}
IDS = list(CASES)

needs_reference = pytest.mark.skipif(not O.have_reference(), reason="the reference build (oracle/_ref, build/librefdecopt.so) is not here")


def _kw(cid):
    _, _, scale, dct, fancy, cs = CASES[cid]
    return dict(scale=scale, dct=dct, fancy=fancy, colorspace=cs, all_scales=True)


def _info(jpeg):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    info = A.SourceInfo()
    A.check(mj._lib.b200jpeg_parse_source(jpeg, len(jpeg), C.byref(info)), "parse_source")
    return info


# ------------------------------------------------------------------------------------------------------------- CPU
def test_golden_covers_every_case():
    assert set(PIX) == set(CASES)
    assert set(YUV) == {Y.case_id(*c) for c in S.YUV_CASES}
    assert {Y.case_id(s, f, "int") for s in S.YUV_SOURCES for f in S.TJ_NEW} <= set(YUV)
    # every block size 1 .. 16 for every layout
    for sid in S.LAYOUT_IDS:
        assert {O.block_size(*CASES[c][2]) for c in CASES if CASES[c][1] == sid} == set(range(1, 17))


@pytest.mark.parametrize("cid", IDS)
def test_size_queries_match_the_reference_and_plan(built, cid):
    import mozjpeg_b200 as mj
    _, sid, scale, dct, fancy, cs = CASES[cid]
    jpeg = O.source(sid)[0]
    want = PIX[cid]
    assert O.md5(jpeg) == want["src_md5"]
    w, h, ocs, onc = mj.decompress_output(_info(jpeg), **_kw(cid))
    assert [h, w] + ([onc] if onc > 1 else []) == want["shape"] and ocs == want["out_color_space"]
    pw, ph, comps = O.plan(_info(jpeg), scale, fancy)
    assert (ph, pw) == tuple(want["shape"][:2])
    assert [list(c[:3]) for c in comps] == want["components"]


@pytest.mark.parametrize("n", S.NEW_SIZES)
def test_matrices_equal_the_restatement(n):
    rng = np.random.default_rng(n)
    coef = rng.integers(-32768, 32768, (512, 64))
    q = rng.integers(0, 65536, (512, 64))
    coef[:32] = 32767; coef[32:64] = -32768; q[:64] = 65535
    coef[64:96] = rng.integers(-1023, 1024, (32, 64)); q[64:96] = 1
    assert (S.idct_scaled(coef, q, n) == S.idct_by_matrix(coef, q, n)).all()


def test_generated_device_functions_are_current():
    sys.path.insert(0, os.path.join(S.ROOT, "tools"))
    import gen_idct_scaled as G
    assert open(G.OUT).read() == G.render()


GRAY = [c for c in IDS if CASES[c][1] in ("o_gray", "idct_q1", "idct_q255", "idct_q32767") and CASES[c][5] is None]


@pytest.mark.parametrize("cid", GRAY)
def test_numpy_idct_gives_the_golden_gray_pixels(cid):
    import recompress_cases as R
    _, sid, scale, _, _, _ = CASES[cid]
    n = O.block_size(*scale)
    if n in (1, 2, 4, 8):
        pytest.skip("jidctred.c / 8x8 sizes are covered by the decompress-options tests")
    jpeg, planes = R.source(sid) if sid.startswith("idct_") else O.source(sid)
    if sid.startswith("idct_"):
        plane, q = planes[0], np.full(64, R.IDCT_TABLES[sid])
    else:
        from oracle import oracle as OR
        try:
            r = OR.ref_read_coefs(jpeg)
        except Exception:
            pytest.skip("the reference build is not here to read the coefficients of an oracle-written source")
        plane, q = r["coefs"][0], r["qt"][0]
    hib, wib = plane.shape[:2]
    blk = S.idct_scaled(plane.reshape(-1, 64), q, n).reshape(hib, wib, n, n).transpose(0, 2, 1, 3).reshape(hib * n, wib * n)
    h, w = PIX[cid]["shape"][:2]
    assert O.md5(np.ascontiguousarray(blk[:h, :w])) == PIX[cid]["pix_md5"]


@needs_reference
@pytest.mark.parametrize("n", S.NEW_SIZES)
def test_numpy_idct_equals_the_reference_on_constructed_blocks(built, n):
    """coefficients at +-1023 (the largest an 8-bit file codes) under tables of 1, 255 and 32767, through a gray file
    the oracle writes"""
    import mozjpeg_b200 as mj
    from oracle import oracle as OR
    rng = np.random.default_rng(100 + n)
    lim = 1023
    for tab in (1, 255, 32767):
        blocks = [np.full(64, lim, np.int16), np.full(64, -lim, np.int16)]
        for k in range(64):
            b = np.zeros(64, np.int16); b[k] = lim if k % 2 else -lim; blocks.append(b)
        blocks += [rng.integers(-lim, lim + 1, 64).astype(np.int16) for _ in range(62)]
        plane = np.stack(blocks).reshape(8, 16, 64)
        p = mj.params_from_switches(["-revert"], 16 * 8, 8 * 8, 1)
        for k in range(64):
            p.quant_tbl[0][k] = tab
        jpeg = OR.oracle_encode_coefs(p, [plane])
        px, _, msg = O.ref_decompress(jpeg, (n, 8, 0, 1, -1))
        assert px is not None, msg
        r = OR.ref_read_coefs(jpeg)
        got = S.idct_scaled(r["coefs"][0].reshape(-1, 64), r["qt"][0], n).reshape(8, 16, n, n).transpose(0, 2, 1, 3).reshape(8 * n, 16 * n)
        assert (got == px).all(), (n, tab)


@pytest.mark.parametrize("scale", [(3, 8), (3, 4), (7, 8), (9, 8), (2, 1), (3, 2)])
def test_without_all_scales_the_message_is_unchanged(built, scale):
    import mozjpeg_b200 as mj
    jpeg = O.source("o_420")[0]
    k = O.block_size(*scale)
    msg = f"scale {scale[0]}/{scale[1]} gives an IDCT block size of {k}: only sizes 1, 2, 4 and 8 (1/8, 1/4, 1/2, 1/1) are decoded on the device"
    with pytest.raises(mj.B200JpegError) as e:
        mj.decompress_output(_info(jpeg), scale=scale)
    assert msg in str(e.value)
    with pytest.raises(mj.B200JpegError) as e:
        mj.decompress_output(_info(jpeg), scale=scale, all_scales=False)
    assert msg in str(e.value)
    mj.decompress_output(_info(jpeg), scale=scale, all_scales=True)
    if scale in S.TJ_NEW:
        y = Y.source("y_420")
        with pytest.raises(mj.B200JpegError):
            mj.decompress_yuv_dims(_info(y), scale=scale)
        ss, dims = mj.decompress_yuv_dims(_info(y), scale=scale, all_scales=True)
        assert [list(d) for d in dims] == YUV[Y.case_id("y_420", scale, "int")]["dims"]


def test_positional_options_keep_working():
    from mozjpeg_b200 import _abi as A
    o = A.DecompressOptions(1, 1, 7, 1, -1)
    assert (o.scale_num, o.scale_denom, o.dct_method, o.do_fancy_upsampling, o.out_color_space, o.all_scales) == (1, 1, 7, 1, -1, 0)


def test_djpeg_parse_leaves_all_scales_to_main():
    from mozjpeg_b200 import djpeg
    assert "all_scales" not in djpeg.parse(["-scale", "3/4"])


@needs_reference
@pytest.mark.gpu
@pytest.mark.parametrize("sid,scale", [("o_420", "3/4"), ("o_gray", "3/8"), ("o_422", "9/8"), ("o_rgb", "2/1")])
def test_djpeg_writes_the_reference_ppm(built, tmp_path, sid, scale):
    """python -m mozjpeg_b200.djpeg -scale M/N against the reference library's pixels at the same scale, framed as
    wrppm.c writes them (P5 / P6, width height, 255, rows)"""
    import subprocess
    src = tmp_path / "in.jpg"
    src.write_bytes(O.source(sid)[0])
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.djpeg", "-scale", scale, str(src)], capture_output=True, cwd=S.ROOT)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    num, denom = map(int, scale.split("/"))
    px, _, msg = O.ref_decompress(src.read_bytes(), (num, denom, 0, 1, -1))
    assert px is not None, msg
    h, w = px.shape[:2]
    want = (b"P5" if px.ndim == 2 else b"P6") + f"\n{w} {h}\n255\n".encode() + px.tobytes()
    assert r.stdout == want


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_every_golden_case_on_the_device(built):
    import mozjpeg_b200 as mj
    import torch
    enc = mj.Encoder(0)
    bad = []
    for cid in IDS:
        jpeg = O.source(CASES[cid][1])[0]
        px = enc.decompress([jpeg], **_kw(cid))[0]
        if O.md5(px) != PIX[cid]["pix_md5"]:
            bad.append(cid)
    assert not bad, bad[:10]
    # device pointers, one case per size
    for k in S.NEW_SIZES:
        cid = O.case_id("o_420", (k, 8), "int", True, None)
        jpeg = O.source("o_420")[0]
        h, w, nc = PIX[cid]["shape"]
        t = torch.zeros((2, h, w, nc), dtype=torch.uint8, device="cuda:0")
        enc.decompress_ptr([jpeg, jpeg], t.data_ptr(), w * nc, h * w * nc, **_kw(cid))
        torch.cuda.synchronize()
        for i in range(2):
            assert O.md5(t[i].cpu().numpy()) == PIX[cid]["pix_md5"], cid
    enc.close()


@pytest.mark.gpu
def test_yuv_planes_at_the_new_factors(built):
    import mozjpeg_b200 as mj
    import torch
    enc = mj.Encoder(0)
    for sid, scale, dct in S.YUV_CASES:
        src = Y.source(sid)
        want = YUV[Y.case_id(sid, scale, dct)]
        planes = enc.decompress_yuv([src, src], scale=scale, dct=dct, all_scales=True)
        _, dims = Y.plan(_info(src), scale)
        for i in range(2):
            assert [Y.md5(Y.defined(p, *d)) for p, d in zip(planes[i], dims)] == want["md5"], (sid, scale, dct)
        # device planes prefilled, at an odd pitch: bytes outside the written region stay
        ts = [torch.full((2, ph + 3, pw + 5), 0xA5, dtype=torch.uint8, device="cuda:0") for pw, ph in want["dims"]]
        enc.decompress_yuv_ptr([src, src], [t.data_ptr() for t in ts], [t.shape[2] for t in ts], [t.shape[1] * t.shape[2] for t in ts],
                               scale=scale, dct=dct, all_scales=True)
        torch.cuda.synchronize()
        for t, d, m in zip(ts, dims, want["md5"]):
            a = t.cpu().numpy()
            pw, ph, iw, ih = d
            cw, ch = min(iw, pw), min(ih, ph)
            for i in range(2):
                assert Y.md5(a[i, :ch, :cw]) == m, (sid, scale, dct)
                outside = a[i].copy(); outside[:ch, :cw] = 0xA5
                assert (outside == 0xA5).all(), (sid, scale, dct)
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 1, 3])
def test_batches_equal_single_calls(built, chunk):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    enc.set_chunk_images(chunk)
    jpeg = O.source("o_420")[0]
    for scale in ((3, 8), (5, 8), (13, 8), (2, 1)):
        kw = dict(scale=scale, all_scales=True)
        one = enc.decompress([jpeg], **kw)[0]
        many = enc.decompress([jpeg] * 5, **kw)
        assert all((m == one).all() for m in many), scale
        y = Y.source("y_422")
        p1 = enc.decompress_yuv([y], **kw)[0]
        pn = enc.decompress_yuv([y] * 4, **kw)
        assert all(all((a == b).all() for a, b in zip(p, p1)) for p in pn), scale
    enc.close()


@pytest.mark.gpu
def test_one_geometry_chunks_count_sample_bytes(built):
    """a 3840x2160 4:2:0 frame is 194,400 blocks: eight share a chunk of the ~1.6 M-block budget at 1/1, two at 2/1
    (16 x 16 samples a block count four times), three at 3/2 (12 x 12: 2.25 times)"""
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    src = O.source("o_4k")[0]
    for kw, want in ((dict(scale=(1, 1)), 5), (dict(scale=(2, 1), all_scales=True), 2), (dict(scale=(3, 2), all_scales=True), 3)):
        out = enc.decompress([src] * 5, **kw)
        assert enc.chunk_images() == want, kw
        assert all((o == out[0]).all() for o in out[1:]), kw
    enc.close()


@pytest.mark.gpu
def test_ladder_through_renditions_equals_single_calls(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    files = [O.source("o_420")[0], O.source("o_420")[0]]
    rungs = [dict(scale=s, all_scales=True) for s in S.LADDER]
    out = enc.decompress_renditions(files, rungs)
    for r, kw in enumerate(rungs):
        single = enc.decompress(files, **kw)
        for i in range(len(files)):
            assert (out[r][i] == single[i]).all(), (r, i)
    rec = []
    for kw, q in zip(rungs, ("80", "75", "70")):
        p = mj.params_for_jpeg_input(["-quality", q], files[0], **kw)
        rec.append((p, kw))
    outs = enc.recompress_renditions(files, rec)
    for r, (p, kw) in enumerate(rec):
        assert outs[r] == enc.recompress(p, files, **kw), r
    enc.close()


@pytest.mark.gpu
def test_mixed_batches_with_scaled_rungs_equal_single_calls(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    files = [O.source(s)[0] for s in ("o_420", "o_gray", "o_422", "o_4k", "o_rgb", "o_440", "o_444")]
    rungs = [dict(scale=(3, 4), all_scales=True), dict(scale=(2, 1), all_scales=True, fancy=False), dict(scale=(5, 8), all_scales=True, dct="fast")]
    out = enc.decompress_mixed(files, rungs)
    for r, kw in enumerate(rungs):
        for i, f in enumerate(files):
            assert (out[r][i] == enc.decompress([f], **kw)[0]).all(), (r, i)
    # a 4K 4:2:0 frame is 194,400 blocks; at 2/1 its sample planes count four times that, so at most two frames share a
    # chunk of the ~1.6 M-block budget (eight at 1/1): chunks [4K, 4K] and [4K, 4K, 227x149], and the outputs still
    # equal the single calls
    four = enc.decompress_mixed([files[3]] * 4 + [files[0]], [dict(scale=(2, 1), all_scales=True)])[0]
    assert enc.chunk_images() == 3
    single = enc.decompress([files[3]], scale=(2, 1), all_scales=True)[0]
    assert all((four[i] == single).all() for i in range(4))
    # one image over the budget at 2/1 though under it in coefficient blocks: 3200x2800 4:4:4 is 420,000 blocks, 1.68 M
    # at 2/1, so it is a chunk of its own between two small files
    from mozjpeg_b200.synth import synth_image
    big = enc.encode_batch(mj.params_from_switches(["-revert", "-quality", "90", "-sample", "1x1"], 3200, 2800), synth_image(5, 3200, 2800)[None])[0]
    trio = [files[0], big, files[1]]
    out = enc.decompress_mixed(trio, [dict(scale=(2, 1), all_scales=True)])[0]
    assert enc.chunk_images() == 1
    for i, f in enumerate(trio):
        assert (out[i] == enc.decompress([f], scale=(2, 1), all_scales=True)[0]).all(), i
    enc.close()


@pytest.mark.gpu
def test_recompress_at_three_quarters_equals_encoding_the_pixels(built):
    import mozjpeg_b200 as mj
    import recompress_cases as R
    jpeg = O.source("o_420")[0]
    kw = dict(scale=(3, 4), all_scales=True)
    p = mj.params_for_jpeg_input(["-quality", "85"], jpeg, **kw)
    enc = mj.Encoder(0)
    out = enc.recompress(p, [jpeg], **kw)[0]
    px = enc.decompress([jpeg], **kw)
    ref = enc.encode_batch(p, px)[0]
    assert out == R.insert_markers(ref, R.copied_markers(jpeg, p))
    enc.close()


@needs_reference
@pytest.mark.gpu
@pytest.mark.parametrize("scale", [(3, 8), (5, 4)])
def test_progressive_sources(built, scale):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    enc.set_progressive_decode(True)
    for sid in Y.PROGRESSIVE:
        src = Y.source(sid)
        want, _, msg = O.ref_decompress(src, (scale[0], scale[1], 0, 1, -1))
        assert want is not None, msg
        assert (enc.decompress([src], scale=scale, all_scales=True)[0] == want).all(), sid
    enc.close()


@pytest.mark.gpu
def test_what_stays_refused_is_refused_the_same_way(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    enc.set_progressive_decode(True)
    for sid in ("prog:cmyk", "prog:prog12", "prog:drop_to_dc_only"):      # 4-component, 12-bit, block smoothing
        src = Y.source(sid)
        with pytest.raises(mj.B200JpegError) as a:
            enc.decompress([src], scale=(1, 1))
        with pytest.raises(mj.B200JpegError) as b:
            enc.decompress([src], scale=(3, 4), all_scales=True)
        assert str(a.value) == str(b.value), sid
    enc.close()
