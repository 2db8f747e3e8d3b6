"""GPU: the default sequential trellis at 8 bits behind the tiled forward kernel counts its statistics in that kernel
(AC symbols from the plain-quantized blocks in shared memory, plain DC values into the dense DC array, then a small DC
statistics kernel) and never writes the plain-quantized coefficient planes.  Checked without B200JPEG_KEEP_PLAIN: the
trellis-phase Huffman tables (built from those statistics) and the files against the CPU oracle, on every sampling layout
of the tiled kernel, ragged sizes (dummy blocks), restarts, the three DCTs, the DC trellis variants, raw-data and
smoothed input, chunked batches on two streams and per-image quantization tables."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def enc(built):
    import mozjpeg_b200 as mj
    assert not os.environ.get("B200JPEG_KEEP_PLAIN")
    e = mj.Encoder(0)
    yield e
    e.close()


def _fused(e):
    st = e.stage_times()
    return "trellis_dc_stats" in st and "trellis_stats" not in st and "dummy" not in st


def _check_tables(e, p, i, dbg):
    for ci in range(p.num_components):
        assert e.debug_huff(i, -1 - ci, False, p.comp_info[ci].dc_tbl_no) == dbg["trellis_dc"][ci], ("dc", i, ci)
        assert e.debug_huff(i, -1 - ci, True, p.comp_info[ci].ac_tbl_no) == dbg["trellis_ac"][ci], ("ac", i, ci)


def _run(e, sw, w, h, n=2, seed=0, fused=True):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    imgs = np.stack([O.synth_image(seed + i, w, h) for i in range(n)])
    p = mj.params_from_switches(sw, w, h)
    out = e.encode_batch(p, imgs)
    assert _fused(e) == fused, (sw, e.stage_times())
    for i in range(n):
        r = O.oracle_encode(p, imgs[i], want_debug=True)
        assert out[i] == r.jpeg, (sw, w, h, i)
        _check_tables(e, p, i, r.dbg)


BASE = ["-baseline", "-quality", "75"]
LAYOUTS = {"gray": ["-grayscale"], "444": ["-sample", "1x1"], "422": ["-sample", "2x1"], "440": ["-sample", "1x2"], "420": ["-sample", "2x2"]}


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("shape", [(128, 64), (203, 141), (9, 17)], ids=lambda s: "%dx%d" % s)
def test_layouts_and_ragged_sizes(enc, layout, shape):
    _run(enc, BASE + LAYOUTS[layout], *shape, seed=11)


@pytest.mark.parametrize("extra", [["-restart", "2"], ["-restart", "7B"], ["-restart", "1B"],
                                   ["-dct", "fast"], ["-dct", "float"], ["-dct", "fast", "-restart", "3B"],
                                   ["-notrellis-dc"], ["-notrellis-dc", "-dct", "float", "-restart", "1"],
                                   ["-trellis-dc-ver-weight", "0.5"], ["-smooth", "30"], ["-quality", "95"], ["-quality", "20"]],
                         ids=lambda s: "_".join(x.lstrip("-") for x in s))
@pytest.mark.parametrize("layout", ["420", "444", "gray"])
def test_switches(enc, extra, layout):
    _run(enc, BASE + LAYOUTS[layout] + extra, 157, 93, seed=21)


def test_generic_forward_layout_keeps_the_statistics_pass(enc):
    """3x2 sampling runs on the one-thread-per-block forward kernel: the separate statistics pass stays."""
    _run(enc, BASE + ["-sample", "3x2"], 100, 61, fused=False)


def test_very_wide_image(enc):
    """Rows too long for the warp-cooperative DC trellis: the fallback kernels write the DC values themselves."""
    _run(enc, BASE + ["-sample", "1x1"], 30000, 16, n=1, seed=77)


def test_extreme_content(enc):
    """Flat, saturated and noisy blocks at quality 100 and 5: the largest plain-quantized values and the longest runs.
    (At 8 bits a plain-quantized AC value needs at most 10 bits and a DC difference at most 11, so the statistics never
    flag JERR_BAD_DCT_COEF here; the check stays for the kernels' sake.)"""
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    rng = np.random.default_rng(9)
    w, h = 96, 80
    imgs = [np.full((h, w, 3), 255, np.uint8), np.zeros((h, w, 3), np.uint8), rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
            (((np.indices((h, w)).sum(0) // 3) % 2) * 255).astype(np.uint8)[..., None].repeat(3, 2)]
    for sw in (BASE[:1] + ["-quality", "100", "-sample", "1x1"], BASE[:1] + ["-quality", "5"], BASE[:1] + ["-quality", "100", "-dct", "float"]):
        p = mj.params_from_switches(sw, w, h)
        out = enc.encode_batch(p, np.stack(imgs))
        assert _fused(enc)
        for i, im in enumerate(imgs):
            r = O.oracle_encode(p, im, want_debug=True)
            assert out[i] == r.jpeg, (sw, i)
            _check_tables(enc, p, i, r.dbg)


def test_raw_data_input(enc):
    import mozjpeg_b200 as mj
    from mozjpeg_b200.synth import synth_planes
    from oracle import oracle as O
    for sw in (BASE + ["-sample", "2x2"], BASE + ["-sample", "1x2", "-dct", "float"], BASE + ["-grayscale", "-restart", "1"]):
        p = mj.params_from_switches(sw, 130, 75, 1 if "-grayscale" in sw else 3)
        per = [synth_planes(p, 60 + i) for i in range(3)]
        out = enc.encode_batch_raw(p, [np.stack([pl[ci] for pl in per]) for ci in range(p.num_components)])
        assert _fused(enc)
        for i in range(3):
            assert out[i] == O.oracle_encode_raw(p, per[i]), (sw, i)


@pytest.mark.parametrize("chunk", [1, 2])
def test_chunks_on_two_streams(built, chunk):
    """Consecutive chunks alternate between two arenas and streams, the last one ragged: each chunk's histograms are
    zeroed on its own stream ahead of its forward kernel."""
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    w, h = 136, 88
    imgs = np.stack([O.synth_image(40 + s, w, h) for s in range(5)])
    p = mj.params_from_switches(BASE + ["-sample", "2x2", "-restart", "1"], w, h)
    e = mj.Encoder(0)
    try:
        e.set_chunk_images(chunk)
        for _ in range(2):
            out = e.encode_batch(p, imgs)
        assert _fused(e)
        for i in range(len(imgs)):
            r = O.oracle_encode(p, imgs[i], want_debug=True)
            assert out[i] == r.jpeg, (chunk, i)
        _check_tables(e, p, len(imgs) - 1, r.dbg)             # the taps hold the last chunk only
    finally:
        e.close()


def test_per_image_tables(enc):
    """Every image's CTAs count into that image's histograms: a mixed-quality batch, and one image at stride 0 under
    several table sets."""
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    w, h = 120, 72
    p = mj.params_from_switches(BASE + ["-sample", "2x2"], w, h)
    qt = mj.quality_tables(p, [30, 75, 92, 50])
    imgs = np.stack([O.synth_image(70 + i, w, h) for i in range(4)])
    for batch in (imgs, imgs[:1]):                            # one image and four table sets: image stride 0
        out = enc.encode_batch(p, batch, qtables=qt)
        assert _fused(enc)
        for i in range(4):
            pi = p.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = qt[i]
            r = O.oracle_encode(pi, batch[i % len(batch)], want_debug=True)
            assert out[i] == r.jpeg, (len(batch), i)
            _check_tables(enc, pi, i, r.dbg)
