"""Sequential Huffman scans packed from code slots (k_block_bits_seq stores each short block's bit string, k_encode_seq
copies it): the device must write the oracle's bytes when the blocks of a tile mix slot blocks and longer (fallback)
blocks, when restart segments end inside tiles, when tiles end mid-word and mid-MCU, on both walk paths (symbol
records behind the trellis, coefficient blocks without it) and in batches with per-image tables."""
import numpy as np
import pytest

BASE = ["-baseline", "-sample", "2x2"]
TWELVE = ["-precision", "12", "-notrellis", "-noovershoot", "-baseline", "-sample", "1x1"]


def _noise(seed, w, h):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _image(kind, seed, w, h):
    from mozjpeg_b200.synth import synth_image, synth_image12
    if kind == "noise":
        return _noise(seed, w, h)
    if kind == "mixed":                          # noise on the left half: dense and sparse blocks in the same tiles
        im = synth_image(seed, w, h)
        im[:, : w // 2] = _noise(seed, w // 2, h)
        return im
    if kind == "synth12":
        return synth_image12(seed, w, h)
    return synth_image(seed, w, h)


CASES = [
    # (image, switches, width, height)
    ("noise", BASE + ["-quality", "95"], 517, 263),
    ("noise", BASE + ["-quality", "100"], 301, 177),
    ("noise", BASE + ["-quality", "98", "-notrellis"], 333, 199),
    ("synth", BASE + ["-quality", "75"], 1003, 517),
    ("mixed", BASE + ["-quality", "75"], 777, 389),
    ("mixed", BASE + ["-quality", "90"], 1921, 91),
    ("synth", BASE + ["-quality", "75", "-restart", "1B"], 611, 307),
    ("mixed", BASE + ["-quality", "75", "-restart", "1B"], 403, 211),
    ("mixed", BASE + ["-quality", "75", "-restart", "7B"], 1001, 301),
    ("noise", BASE + ["-quality", "95", "-restart", "7B"], 269, 131),
    ("mixed", BASE + ["-quality", "75", "-restart", "1"], 833, 263),
    ("mixed", BASE + ["-quality", "85", "-restart", "3"], 509, 381),
    ("mixed", ["-baseline", "-quality", "75", "-grayscale"], 1011, 403),
    ("mixed", ["-baseline", "-quality", "75", "-grayscale", "-notrellis", "-restart", "5B"], 997, 211),
    ("mixed", ["-baseline", "-quality", "80", "-sample", "1x1", "-notrellis"], 701, 333),
    ("noise", ["-baseline", "-quality", "97", "-sample", "1x1", "-notrellis", "-restart", "2"], 259, 137),
    ("synth12", TWELVE + ["-quality", "75"], 643, 271),
    ("synth12", TWELVE + ["-quality", "95", "-restart", "4B"], 389, 157),
]


def _id(c):
    return "%s:%dx%d:%s" % (c[0], c[2], c[3], "_".join(s.lstrip("-") for s in c[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=_id)
def test_slot_packer_matches_oracle(encoder, c):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    kind, sw, w, h = c
    im = _image(kind, 7, w, h)
    p = mj.params_from_switches(sw, w, h)
    ref = O.oracle_encode(p, im).jpeg
    out = encoder.encode_batch(mj.params_from_switches(sw, w, h), im[None])[0]
    assert out == ref


@pytest.mark.gpu
@pytest.mark.parametrize("restart", [[], ["-restart", "3B"]], ids=["plain", "restart3B"])
def test_slot_packer_batch_per_image_tables(encoder, restart):
    """Five images of one batch, each with its own quality's tables and so its own optimal Huffman tables and slot
    widths: image i must be the file the oracle writes for image i alone."""
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    w, h = 645, 331
    qs = [30, 75, 90, 97, 100]
    ims = np.stack([_image("mixed", 20 + i, w, h) for i in range(len(qs))])
    ps = [mj.params_from_switches(BASE + ["-quality", str(q)] + restart, w, h) for q in qs]
    qt = np.stack([np.ctypeslib.as_array(p.quant_tbl).copy() for p in ps])
    outs = encoder.encode_batch(ps[0], ims, qtables=qt)
    for i, p in enumerate(ps):
        assert outs[i] == O.oracle_encode(p, ims[i]).jpeg, "image %d (quality %d)" % (i, qs[i])
