"""The sequential AC trellis groups blocks by their plain-quantized non-zero count inside tiles of consecutive blocks
(k_trellis_ac3<15>, T3_TILE blocks of one image and component): blocks with at most 15 non-zero ACs run in the tile,
blocks with 16..32 and with more than 32 go to per-(image, component) lists that two more kernels run.  These cases
put that split where it can go wrong: components whose block count is not a multiple of the tile, images smaller than
one tile, tiles of all-zero blocks, tiles where every block has more than 32 entries, the class edges 15/16 and 32/33
side by side, per-image tables that move the class mix from image to image, a batch of many images, and the
progressive path, where the trellis writes the block's non-zero mask back into its record.

CPU tests: each case reaches its class mix (the restatement's plain-coefficient tap), and the restatement
(oracle/jpeg_oracle.c) writes the unmodified reference's bytes on it (skipped without oracle/_ref).
GPU tests: the device writes the restatement's bytes."""
import os
import tempfile

import numpy as np
import pytest

import adversarial_cases as AC

SEQ = ["-baseline", "-quality", "75", "-sample", "2x2"]
PROG = ["-fastcrush", "-quality", "75", "-sample", "2x2"]
EDGE_COUNTS = (0, 1, 8, 9, 14, 15, 16, 17, 31, 32, 33, 34, 63)
PER_IMAGE_Q = (30, 95, 85)


def _need_ref():
    from oracle import oracle as O
    if not O.ref_available():
        pytest.skip("oracle/_ref not built")


def _params(sw, img):
    import mozjpeg_b200 as mj
    nc = 1 if img.ndim == 2 else img.shape[2]
    return mj.params_from_switches(sw, img.shape[1], img.shape[0], nc)


def _synth(seed, w, h):
    from mozjpeg_b200.synth import synth_image
    return synth_image(seed, w, h)


def _noise(seed, w, h):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _edge_image(seed=0, wb=40, hb=30):
    """Gray image of basis blocks with exactly the non-zero counts EDGE_COUNTS (values +-1 under a flat table of 16),
    in a seeded random order so that every tile mixes the three classes."""
    rng = np.random.default_rng(seed)
    counts = rng.permutation(np.resize(np.array(EDGE_COUNTS), wb * hb))
    blocks = []
    for n in counts:
        z = np.zeros(64)
        z[rng.choice(np.arange(1, 64), n, replace=False)] = rng.choice([-1, 1], n)
        blocks.append(AC.basis_block(z, 16))
    return AC._blocks_to_image(np.stack(blocks), wb)


EDGE_TABLES = AC.flat_tables([16])[0]

# name -> (switches, images, flat table of 16 or None).  Block counts per component (luma, chroma at 2x2):
#   small  25x17 = 425 and 13x9 = 117, less than one tile
#   ragged 129x65 = 8385 and 65x33 = 2145, 16 and 4 whole tiles and a partial one
CASES = {
    "small": (SEQ, lambda: [_synth(11, 200, 136)], None),
    "ragged": (SEQ, lambda: [_synth(12 + i, 1030, 520) for i in range(2)], None),
    "flat": (["-baseline", "-quality", "75", "-sample", "1x1"], lambda: [np.full((256, 320, 3), 128, np.uint8)], None),
    "noise_q95": (["-baseline", "-quality", "95", "-sample", "1x1"], lambda: [_noise(13, 264, 200)], None),
    "class_edges": (["-baseline"], lambda: [_edge_image()], EDGE_TABLES),
    "progressive_ragged": (PROG, lambda: [_synth(14, 1030, 520)], None),
    "progressive_noise_q95": (["-fastcrush", "-quality", "95", "-sample", "1x1"], lambda: [_noise(15, 264, 200)], None),
    "progressive_class_edges": (["-fastcrush"], lambda: [_edge_image(1)], EDGE_TABLES),
}


def _case_params(name, img):
    sw, _, t = CASES[name]
    p = _params(sw, img)
    if t is not None:
        p = p.copy()
        np.ctypeslib.as_array(p.quant_tbl)[:] = t
    return p


def _ref_bytes(name, img):
    from oracle import oracle as O
    sw, _, t = CASES[name]
    if t is None:
        return O._ref_cjpeg_pixels(img, sw)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "q.txt")
        with open(path, "w") as f:
            for _ in range(4):
                f.write(" ".join(str(int(v)) for v in t.reshape(-1)[:64]) + "\n")      # flat: natural and zigzag order agree
        return O._ref_cjpeg_pixels(img, sw + ["-qtables", path])


def _classes(p, img):
    """Per component: the blocks' plain-quantized non-zero AC counts."""
    from oracle import oracle as O
    d = O.oracle_encode(p, img, want_debug=True).dbg
    return [AC.nonzero_ac_counts(d["plain"][ci][:d["hib"][ci], :d["wib"][ci]]) for ci in range(d["ncomp"])]


def _per_image(sw):
    """Image 0's parameters and the (N, 4, 64) tables of the per-image-quality batch."""
    import mozjpeg_b200 as mj
    img = _synth(20, 640, 400)
    ps = [mj.params_from_switches(sw + ["-quality", str(q)], img.shape[1], img.shape[0], 3) for q in PER_IMAGE_Q]
    return ps, np.stack([np.ctypeslib.as_array(p.quant_tbl).copy() for p in ps]), img


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_cases_reach_their_class_mix(built):
    def nz(name):
        img = CASES[name][1]()[0]
        return _classes(_case_params(name, img), img)
    small, ragged = nz("small"), nz("ragged")
    assert len(small[0]) < 512 and len(small[1]) < 512
    assert all(len(c) % 512 for c in ragged) and all(len(c) > 2048 for c in ragged)
    assert all((c == 0).all() for c in nz("flat"))
    assert all((c > 32).all() for c in nz("noise_q95"))
    assert set(nz("class_edges")[0]) == set(EDGE_COUNTS)
    # every class is present in the ragged luma plane
    y = ragged[0]
    assert (y <= 15).any() and ((y >= 16) & (y <= 32)).any() and (y > 32).any()


def test_per_image_tables_move_the_class_mix(built):
    ps, _, img = _per_image(SEQ)
    shares = [(_classes(p, img)[0] >= 16).mean() for p in ps]
    assert shares[0] < 0.05 and shares[1] > 0.9 and shares[0] < shares[2] < shares[1]


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference(built, name):
    _need_ref()
    from oracle import oracle as O
    for img in CASES[name][1]():
        assert O.oracle_encode(_case_params(name, img), img).jpeg == _ref_bytes(name, img)


@pytest.mark.parametrize("sw", [SEQ, PROG], ids=["baseline", "fastcrush"])
def test_oracle_matches_reference_per_image_quality(built, sw):
    _need_ref()
    from oracle import oracle as O
    ps, _, img = _per_image(sw)
    for p, q in zip(ps, PER_IMAGE_Q):
        assert O.oracle_encode(p, img).jpeg == O._ref_cjpeg_pixels(img, sw + ["-quality", str(q)]), q


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_oracle(encoder, name):
    from oracle import oracle as O
    imgs = CASES[name][1]()
    p = _case_params(name, imgs[0])
    out = encoder.encode_batch(p, np.stack(imgs))
    for i, img in enumerate(imgs):
        assert out[i] == O.oracle_encode(p, img).jpeg, (name, i)


@pytest.mark.gpu
@pytest.mark.parametrize("sw", [SEQ, PROG], ids=["baseline", "fastcrush"])
def test_device_per_image_quality(encoder, sw):
    from oracle import oracle as O
    ps, qt, img = _per_image(sw)
    out = encoder.encode_batch(ps[0], np.stack([img] * len(ps)), qtables=qt)
    for i, p in enumerate(ps):
        assert out[i] == O.oracle_encode(p, img).jpeg, PER_IMAGE_Q[i]


@pytest.mark.gpu
def test_device_batch_of_48(encoder):
    """48 images of 1030x520 in one call: 144 (image, component) rows of tiles, each with its own list counters."""
    from oracle import oracle as O
    base = [_synth(30 + i, 1030, 520) for i in range(4)]
    p = _params(SEQ, base[0])
    out = encoder.encode_batch(p, np.stack([base[i % 4] for i in range(48)]))
    want = [O.oracle_encode(p, b).jpeg for b in base]
    for i in range(48):
        assert out[i] == want[i % 4], i

