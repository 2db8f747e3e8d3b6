"""Batches of mixed geometry: Encoder.decompress_mixed / recompress_mixed (b200jpeg_decompress_mixed /
b200jpeg_recompress_mixed) take files of different sizes, sampling layouts, colour spaces, tables, restart intervals and
sequential / progressive coding in one call.  Every output must be byte for byte what the one-file call makes of that
file with the same options (and params); the existing goldens pin those to the reference.  Where the reference build
exists, a subset is also compared with the reference's decompressor and cjpeg directly.

Every source is written here by the CPU oracle (or, for the one image larger than a chunk's block budget, by the device
encoder), from the case modules' seeded pixels."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import common  # noqa: F401,E402  (puts the repository root on sys.path)
import decode_cases as D  # noqa: E402
import decompress_options_cases as O  # noqa: E402
import recompress_cases as R  # noqa: E402

# (cjpeg switches, decompress options): scales 1/8 .. 1/1, all three IDCT methods, fancy on and off, output colour spaces
LADDER = [
    (["-baseline", "-quality", "80"], {}),
    (["-quality", "75"], dict(scale=(1, 2), dct="fast")),
    (["-revert", "-progressive", "-quality", "70"], dict(scale=(1, 4), dct="float", fancy=False, colorspace="bgrx")),
    (["-baseline", "-quality", "60"], dict(scale=(1, 8), colorspace="gray")),
    (["-quality", "85"], dict(dct="float", fancy=False)),
    (["-baseline", "-quality", "90"], dict(scale=(1, 2), colorspace="xrgb")),
]
LAYOUT_SWITCHES = {lay[0]: lay[4] for lay in O.LAYOUTS}          # gray, 4:4:4, 4:2:2, 4:4:0, 4:2:0, RGB-coded
SMALL = [(1, 1), (7, 9), (17, 33), (1000, 1)]

_cache = {}


def _src(sid, w, h, seed, sw, layout=None):
    key = (sid, w, h, seed, tuple(sw), layout)
    if key not in _cache:
        _cache[key] = D.source((sid, w, h, seed, list(sw), layout))[0]
    return _cache[key]


def mixed_sources():
    """every layout at every small size, the six 227x149 layout sources and one 3840x2160 4:2:0 frame"""
    files = []
    for k, (sid, sw) in enumerate(LAYOUT_SWITCHES.items()):
        for j, (w, h) in enumerate(SMALL):
            files.append(_src(sid, w, h, 100 + 7 * k + j, sw))
        files.append(O.source(sid)[0])
    files.append(O.source("o_4k")[0])
    return files


def content_sources():
    """sequential and progressive files with different restart intervals, Huffman and quantization tables and scan
    layouts (progressive decode on)"""
    return [
        _src("p_444", 300, 200, 11, ["-quality", "85", "-sample", "1x1"]),
        _src("p_420", 131, 77, 12, ["-quality", "70"]),
        _src("p_gray", 90, 61, 13, ["-quality", "92", "-grayscale"]),
        _src("r1_420", 227, 149, 14, ["-revert", "-restart", "1", "-quality", "60"]),
        _src("r3b_422", 160, 100, 15, ["-revert", "-restart", "3B", "-sample", "2x1", "-quality", "95"]),
        _src("opt_444", 99, 101, 16, ["-revert", "-optimize", "-sample", "1x1", "-quality", "50"]),
        _src("multi_420", 64, 48, 17, ["-revert", "-quality", "80"], "multi"),
        _src("rprog", 120, 90, 18, ["-revert", "-progressive", "-restart", "2", "-quality", "75"]),
    ]


def _err(fn):
    import mozjpeg_b200 as mj
    with pytest.raises(mj.B200JpegError) as e:
        fn()
    return e.value


def _single_pixels(encoder, f, kw):
    return encoder.decompress([f], **kw)[0]


def _no_encoder():
    import mozjpeg_b200 as mj
    return mj.Encoder.__new__(mj.Encoder)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_python_arguments_are_checked_before_any_call(built):
    import mozjpeg_b200 as mj
    enc = _no_encoder()
    jpeg = O.source("o_420")[0]
    for bad in ([], [dict(sclae=(1, 2))], [(1, 2)]):
        with pytest.raises(ValueError):
            enc.decompress_mixed([jpeg], bad)
        with pytest.raises(ValueError):
            enc.recompress_mixed([jpeg], [([], kw) for kw in bad] if bad and isinstance(bad[0], dict) else bad)
    with pytest.raises(ValueError, match="2 pointers"):
        enc.decompress_mixed_ptr([jpeg, jpeg], [{}], [0], [0])
    p = mj.params_for_jpeg_input([], jpeg)
    for bad in ([("-quality", {})], [("-quality 80", {})], [([], [])], [(p, {})]):
        with pytest.raises(ValueError):
            enc.recompress_mixed([jpeg], bad)
    with pytest.raises(ValueError, match="2 Params"):
        enc.recompress_mixed_params([jpeg, jpeg], [([p], {})])


def test_the_mixed_sources_differ_in_geometry(built):
    from mozjpeg_b200 import jpegtran as T
    geoms = set()
    for f in mixed_sources():
        s = T.parse_source(f)
        geoms.add((s.image_width, s.image_height, s.num_components, s.jpeg_color_space,
                   tuple((s.h_samp_factor[c], s.v_samp_factor[c]) for c in range(s.num_components))))
    assert len(geoms) == len(mixed_sources())


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_decompress_mixed_equals_the_single_calls(encoder):
    files = mixed_sources()
    opts = [kw for _, kw in LADDER]
    out = encoder.decompress_mixed(files, opts)
    assert len(out) == len(opts) and all(len(row) == len(files) for row in out)
    for r, kw in enumerate(opts):
        for i, f in enumerate(files):
            single = _single_pixels(encoder, f, kw)
            assert out[r][i].shape == single.shape and np.array_equal(out[r][i], single), (r, i)
    default = encoder.decompress_mixed(files)
    assert len(default) == 1
    for i, f in enumerate(files):
        assert np.array_equal(default[0][i], encoder.decompress([f])[0]), i


@pytest.mark.gpu
def test_recompress_mixed_equals_the_single_calls(encoder):
    import mozjpeg_b200 as mj
    files = mixed_sources()
    out = encoder.recompress_mixed(files, LADDER)
    for r, (sw, kw) in enumerate(LADDER):
        for i, f in enumerate(files):
            single = encoder.recompress(mj.params_for_jpeg_input(sw, f, **kw), [f], **kw)[0]
            assert out[r][i] == single, (r, i)
    # the explicit-params form, and outputs readable through get_output in rung-major order
    rungs = [([mj.params_for_jpeg_input(sw, f, **kw) for f in files], kw) for sw, kw in LADDER[:2]]
    again = encoder.recompress_mixed_params(files, rungs)
    assert again == out[:2]
    assert encoder.get_output(len(files) + 3) == out[1][3]


@pytest.mark.gpu
def test_mixed_content_sequential_and_progressive(encoder):
    import mozjpeg_b200 as mj
    files = content_sources() + mixed_sources()[::5]
    encoder.set_progressive_decode(True)
    try:
        opts = [{}, dict(scale=(1, 2), dct="fast", colorspace="rgbx"), dict(scale=(1, 4), fancy=False)]
        out = encoder.decompress_mixed(files, opts)
        for r, kw in enumerate(opts):
            for i, f in enumerate(files):
                assert np.array_equal(out[r][i], _single_pixels(encoder, f, kw)), (r, i)
        ladder = [(["-quality", "80"], {}), (["-revert", "-baseline", "-quality", "75"], dict(scale=(1, 4)))]
        rec = encoder.recompress_mixed(files, ladder)
        for r, (sw, kw) in enumerate(ladder):
            for i, f in enumerate(files):
                assert rec[r][i] == encoder.recompress(mj.params_for_jpeg_input(sw, f, **kw), [f], **kw)[0], (r, i)
    finally:
        encoder.set_progressive_decode(False)


@pytest.mark.gpu
def test_permuting_the_inputs_permutes_the_outputs(encoder):
    files = mixed_sources()[:-1]
    opts = [{}, dict(scale=(1, 2))]
    out = encoder.decompress_mixed(files, opts)
    perm = np.random.default_rng(3).permutation(len(files))
    pout = encoder.decompress_mixed([files[j] for j in perm], opts)
    for r in range(len(opts)):
        for k, j in enumerate(perm):
            assert np.array_equal(pout[r][k], out[r][j])
    rec = encoder.recompress_mixed(files, LADDER[:2])
    prec = encoder.recompress_mixed([files[j] for j in perm], LADDER[:2])
    for r in range(2):
        assert prec[r] == [rec[r][j] for j in perm]


@pytest.mark.gpu
def test_a_uniform_batch_gives_the_batch_routes_outputs(encoder):
    import mozjpeg_b200 as mj
    files = [_src("u_420", 227, 149, 30 + k, ["-revert", "-sample", "2x2", "-quality", str(60 + 10 * k)]) for k in range(3)]

    def launches(fn):
        before = encoder.kernel_launches()
        got = fn()
        return got, encoder.kernel_launches() - before
    for kw in [{}, dict(scale=(1, 2), dct="float"), dict(colorspace="gray")]:
        out, n_mixed = launches(lambda: encoder.decompress_mixed(files, [kw])[0])
        rend, n_rend = launches(lambda: encoder.decompress_renditions(files, [kw])[0])
        batch, n_batch = launches(lambda: encoder.decompress(files, **kw))
        assert all(np.array_equal(out[i], batch[i]) and np.array_equal(rend[i], batch[i]) for i in range(len(files))), kw
        assert n_mixed == n_rend == n_batch, (kw, n_mixed, n_rend, n_batch)
    p = mj.params_for_jpeg_input(["-quality", "75"], files[0])
    assert encoder.recompress_mixed(files, [(["-quality", "75"], {})])[0] == encoder.recompress(p, files)


@pytest.mark.gpu
def test_chunking(encoder):
    import mozjpeg_b200 as mj
    files = mixed_sources()[:-1]
    opts = [{}, dict(scale=(1, 4), dct="fast")]
    want = encoder.decompress_mixed(files, opts)
    assert encoder.chunk_images() == len(files)                  # far below the block budget: one chunk
    try:
        for c in (1, 3):
            encoder.set_chunk_images(c)
            got = encoder.decompress_mixed(files, opts)
            assert encoder.chunk_images() == c
            assert all(np.array_equal(got[r][i], want[r][i]) for r in range(2) for i in range(len(files))), c
    finally:
        encoder.set_chunk_images(0)
    # one image above the ~1.6 M-block budget (6000 x 6000 4:4:4, 1.69 M blocks) forms a chunk of its own
    w = h = 6000
    y, x = np.mgrid[0:h, 0:w]
    px = np.stack([(x * 255 // w), (y * 255 // h), ((x + y) * 7 & 255)], axis=-1).astype(np.uint8)
    big = encoder.encode_batch(mj.params_from_switches(["-revert", "-sample", "1x1", "-quality", "50"], w, h, 3), px[None])[0]
    del px
    small = files[:2]
    got = encoder.decompress_mixed([small[0], big, small[1]], [dict(scale=(1, 8))])[0]
    assert encoder.chunk_images() == 1
    for g, f in zip(got, [small[0], big, small[1]]):
        assert np.array_equal(g, _single_pixels(encoder, f, dict(scale=(1, 8))))


@pytest.mark.gpu
def test_launches_do_not_grow_with_the_geometries(encoder):
    uniform = [_src("l_420", 227, 149, 40 + k, ["-revert"]) for k in range(3)]
    mixed = [O.source("o_420")[0], O.source("o_444")[0], _src("l_422", 301, 17, 43, ["-revert", "-sample", "2x1"])]
    counts = []
    for files in (uniform, mixed):
        before = encoder.kernel_launches()
        encoder.decompress_mixed(files)
        counts.append(encoder.kernel_launches() - before)
    assert counts[0] == counts[1]
    # the decode's six stages once, three IDCT launches (one per component slot) and one upsampling launch
    assert counts[1] == 6 + 3 + 1


def _check_refusal(encoder, fn, code, words):
    e = _err(fn)
    assert e.code == code and all(w in str(e) for w in words), str(e)
    return e


@pytest.mark.gpu
def test_refusals(encoder):
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O2
    good = mixed_sources()[:6]
    k = 3
    bad_marker = good[0][:2] + b"\xff\x02" + good[0][4:]                     # an unknown marker where APP0 was
    prog = O2.oracle_encode(mj.params_from_switches(["-progressive", "-revert"], 200, 136, 3), D.pixels(3, 200, 136)).jpeg
    s32 = D.source(next(c for c in D.CASES if c[0] == "sample_3x2"))[0]
    refused = [(bad_marker, A.ERR_BAD_SOURCE, "unknown JPEG marker"), (prog, A.ERR_UNSUPPORTED, "progressive"),
               (D.extra_source("baseline12"), A.ERR_UNSUPPORTED, "12-bit"), (D.extra_source("cmyk"), A.ERR_UNSUPPORTED, "4-component"),
               (s32, A.ERR_UNSUPPORTED, "sampling")]
    for f, code, word in refused:
        single = _err(lambda: encoder.decompress([f]))
        assert single.code == code and word in str(single), str(single)
        files = good[:k] + [f] + good[k:]
        before = encoder.kernel_launches()
        _check_refusal(encoder, lambda: encoder.decompress_mixed(files, [{}, dict(scale=(1, 2))]), code, [f"image {k}:", word])
        _check_refusal(encoder, lambda: encoder.recompress_mixed(files, LADDER[:2]), code, [f"image {k}:", word])
        assert encoder.kernel_launches() == before
    # refused rung options: for every image (a scale off the device's block sizes) and for one image only (CMYK output
    # is refused; gray output of an RGB-coded file is not, YCbCr output of a gray file is)
    before = encoder.kernel_launches()
    _check_refusal(encoder, lambda: encoder.decompress_mixed(good, [{}, dict(scale=(3, 8))]), A.ERR_UNSUPPORTED, ["rendition 1:"])
    gray_at = next(i for i, f in enumerate(mixed_sources()) if T.parse_source(f).num_components == 1 and i > 0)
    files = [mixed_sources()[6]] + [mixed_sources()[gray_at]]
    _check_refusal(encoder, lambda: encoder.decompress_mixed(files, [dict(colorspace="ycbcr")]), A.ERR_PARAM, ["rendition 0, image 1:"])
    # a parameter block that does not describe one image's decoded size, colour space or components
    ps = [mj.params_for_jpeg_input(["-quality", "80"], f) for f in good]
    ps[4] = mj.params_for_jpeg_input(["-quality", "80"], good[0])
    _check_refusal(encoder, lambda: encoder.recompress_mixed_params(good, [(ps, {})]), A.ERR_PARAM, ["rendition 0, image 4:", "decodes to"])
    ps2 = [mj.params_for_jpeg_input([], f, scale=(1, 2)) for f in good]            # image 0 (1x1) decodes to 1x1 at both scales
    _check_refusal(encoder, lambda: encoder.recompress_mixed_params(good, [(ps2, dict(scale=(1, 2))), (ps2, {})]), A.ERR_PARAM, ["rendition 1, image 1:"])
    assert encoder.kernel_launches() == before
    # corrupt entropy-coded data shows in the decode, names the image, and the encoder carries on
    sc = T.parse_source(good[5]).scans[0]
    truncated = good[5][:sc.data_offset + sc.data_size // 2]
    _check_refusal(encoder, lambda: encoder.decompress_mixed(good[:2] + [truncated], [{}]), A.ERR_BAD_SOURCE, ["image 2:", "corrupt"])
    out = encoder.decompress_mixed(good, [{}])[0]
    assert all(np.array_equal(out[i], encoder.decompress([f])[0]) for i, f in enumerate(good))


@pytest.mark.gpu
def test_device_pointers(encoder):
    import torch
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    files = mixed_sources()[:8]
    opts = [{}, dict(scale=(1, 2), colorspace="bgrx")]
    want = encoder.decompress_mixed(files, opts)
    bufs, ptrs, pitch = [], [], []
    for r, kw in enumerate(opts):
        for i, f in enumerate(files):
            w, h, _, nc = mj.decompress_output(T.parse_source(f), **kw)
            p = (w * nc + 31) // 32 * 32 + 32                     # a pitch wider than the row
            t = torch.full((h, p), 7, dtype=torch.uint8, device="cuda")
            bufs.append((t, w * nc)); ptrs.append(t.data_ptr()); pitch.append(p)
    encoder.decompress_mixed_ptr(files, opts, ptrs, pitch)
    torch.cuda.synchronize()
    for j, (t, row) in enumerate(bufs):
        r, i = divmod(j, len(files))
        a = t.cpu().numpy()
        assert np.array_equal(a[:, :row].reshape(want[r][i].shape), want[r][i]), (r, i)
        assert (a[:, row:] == 7).all()


needs_reference = pytest.mark.skipif(not (O.have_reference() and R.have_reference()),
                                     reason="the reference build (oracle/_ref, build/librefdecopt.so, build/librefdec.so) is not here")


@pytest.mark.gpu
@needs_reference
def test_a_subset_equals_the_reference(encoder):
    import mozjpeg_b200 as mj
    files = mixed_sources()[::4]
    opts = [kw for _, kw in LADDER[:4]]
    out = encoder.decompress_mixed(files, opts)
    for r, kw in enumerate(opts):
        o = O.opts_tuple(kw.get("scale", (1, 1)), kw.get("dct", "int"), kw.get("fancy", True), kw.get("colorspace"))
        for i, f in enumerate(files):
            ref, _, msg = O.ref_decompress(f, o)
            assert ref is not None, msg
            assert np.array_equal(out[r][i], ref), (r, i)
    rec = encoder.recompress_mixed(files, LADDER[:1])
    for i, f in enumerate(files):
        assert rec[0][i] == R.ref_cjpeg(f, LADDER[0][0]), i
