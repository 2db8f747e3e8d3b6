"""GPU: every scan is byte-stuffed in one pass (k_stuff: each 4096-byte tile counts its 0xFF bytes, takes its output
offset from a decoupled look-back over the tiles before it, and stores its stuffed bytes from shared memory).  The files
are compared with the CPU oracle on sequential scans from symbol records and from coefficient blocks (also at 12 bits),
streams of one tile and of many, restart markers (whose 0xFF is not stuffed) at every interval kind, streams full of
0xFF bytes whose first call overflows the output buffer (the host retries), chunked batches on two streams, per-image
tables, and the progressive coder and the scan search."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def enc(built):
    import mozjpeg_b200 as mj
    e = mj.Encoder(0)
    yield e
    e.close()


def _check(e, sw, imgs):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    h, w = imgs.shape[1:3]
    p = mj.params_from_switches(sw, w, h)
    out = e.encode_batch(p, imgs)
    assert "stuff" in e.stage_times()
    for i in range(len(imgs)):
        assert out[i] == O.oracle_encode(p, imgs[i]).jpeg, (sw, w, h, i)


def _synth(n, w, h, seed):
    from oracle import oracle as O
    return np.stack([O.synth_image(seed + i, w, h) for i in range(n)])


BASE = ["-baseline", "-quality", "75"]
LAYOUTS = {"gray": ["-grayscale"], "444": ["-sample", "1x1"], "420": ["-sample", "2x2"], "3x2": ["-sample", "3x2"]}


@pytest.mark.parametrize("trellis", [[], ["-notrellis"]], ids=["trellis", "notrellis"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts(enc, layout, trellis):
    _check(enc, BASE + LAYOUTS[layout] + trellis, _synth(2, 203, 141, 5))


def test_twelve_bit(enc):
    from mozjpeg_b200.synth import synth_image12
    imgs = np.stack([synth_image12(7 + i, 72, 40) for i in range(2)])
    _check(enc, ["-precision", "12", "-quality", "75", "-notrellis", "-noovershoot", "-baseline", "-sample", "1x1"], imgs)


# gray: one block per MCU, so the scan's block count is the image's block count
@pytest.mark.parametrize("shape", [(64, 64), (128, 128), (2056, 8), (8, 2056), (1040, 72)],
                         ids=["one_tile", "256_blocks", "257_blocks_row", "257_blocks_column", "many_tiles"])
@pytest.mark.parametrize("trellis", [[], ["-notrellis"]], ids=["trellis", "notrellis"])
def test_tile_counts(enc, shape, trellis):
    _check(enc, BASE + ["-grayscale"] + trellis, _synth(2, *shape, 13))


@pytest.mark.parametrize("restart", [["-restart", "1B"], ["-restart", "1"], ["-restart", "300B"], ["-restart", "128B"], ["-restart", "43B"]],
                         ids=["1B", "1row", "longer_than_a_tile", "ends_on_tile_end", "43B"])
@pytest.mark.parametrize("layout", ["gray", "420"])
@pytest.mark.parametrize("trellis", [[], ["-notrellis"]], ids=["trellis", "notrellis"])
def test_restarts(enc, restart, layout, trellis):
    _check(enc, BASE + LAYOUTS[layout] + trellis + restart, _synth(2, 1040, 72, 17))


def test_output_overflow_retry(built):
    """Noise at quality 100 in 4:4:4: the first call's output buffer (16 bytes per block + 64 KB) is too small, so the
    host retries with a larger one."""
    import mozjpeg_b200 as mj
    rng = np.random.default_rng(3)
    imgs = rng.integers(0, 256, (2, 160, 256, 3), dtype=np.uint8)
    for sw in (["-baseline", "-quality", "100", "-sample", "1x1"], ["-baseline", "-quality", "100", "-sample", "1x1", "-notrellis", "-restart", "5B"]):
        e = mj.Encoder(0)                                      # a fresh encoder starts from the small buffers
        try:
            _check(e, sw, imgs)
        finally:
            e.close()


@pytest.mark.parametrize("chunk", [1, 2])
def test_chunks_on_two_streams(built, chunk):
    """Consecutive chunks alternate between two arenas and streams: each chunk clears its own look-back state."""
    import mozjpeg_b200 as mj
    e = mj.Encoder(0)
    try:
        e.set_chunk_images(chunk)
        for _ in range(2):
            _check(e, BASE + ["-sample", "2x2", "-restart", "1"], _synth(5, 136, 88, 40))
    finally:
        e.close()


def test_per_image_tables(enc):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    w, h = 120, 72
    p = mj.params_from_switches(BASE + ["-sample", "2x2"], w, h)
    qt = mj.quality_tables(p, [30, 75, 92, 50])
    imgs = _synth(4, w, h, 70)
    out = enc.encode_batch(p, imgs, qtables=qt)
    assert "stuff" in enc.stage_times()
    for i in range(4):
        pi = p.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = qt[i]
        assert out[i] == O.oracle_encode(pi, imgs[i]).jpeg, i


@pytest.mark.parametrize("sw", [["-quality", "75", "-fastcrush", "-restart", "2B"], ["-quality", "75"]], ids=["progressive", "scan_search"])
def test_progressive_and_scan_search(enc, sw):
    _check(enc, sw, _synth(2, 157, 93, 29))
