"""The sequential scan packer (k_block_bits_seq's code slots, k_scan_layout's offsets, k_encode_seq's slot copies and
fallback walks) at the boundaries of its rules: placed block lengths (6, 31..33, 63..65, 95..97, 127..129 bits and the
128-bit slot at all 32 word phases), fallback blocks first and last in a tile and between slot blocks inside one word,
tiles that end on and inside a word, tiles of 256 slot and of 256 fallback blocks, last tiles of 1 and 255 blocks,
restart segments of one block and slot-sized blocks that end a segment, every padding length, and 0xFF bytes at word
ends, tile edges and in front of markers (tests/seq_pack_cases.py names and finds them).

CPU tests: the serial model of the packed layout writes the oracle's scan bytes on every case, every boundary class is
reached on the walk that names it, and the oracle writes the unmodified reference jpegtran's bytes on the placed
coefficient cases (skipped without oracle/_ref).
GPU tests: the device writes the oracle's file on every case (a mismatch names the first differing byte's block, tile,
word and class), the device's coefficient files decode back to their input planes, and batches that mix an all-slot
and an all-fallback image write each image's own file at every chunking."""
import os
import tempfile

import numpy as np
import pytest

import seq_pack_cases as S

WALKS = sorted(S.WALK_CLASSES)


def _walk_cases(walk):
    return [c for c in S.ALL_CASES if S.case_walk(c) == walk]


@pytest.fixture(scope="module")
def models(built):
    """case id -> the model's scans of the oracle's file"""
    out = {}

    def get(cid):
        if cid not in out:
            f, pl, _ = S.case(cid)
            out[cid] = S.model_scans(f, pl)
        return out[cid]
    return get


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the model pins the layout, every class is reached
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", S.ALL_CASES)
def test_model_writes_the_oracle_scan_bytes(models, cid):
    f, _, _ = S.case(cid)
    scans = models(cid)
    want = S.scan_bytes(f)
    assert len(scans) == len(want)
    for s, w in zip(scans, want):
        if s.data != w:
            i = next((i for i in range(min(len(s.data), len(w))) if s.data[i] != w[i]), min(len(s.data), len(w)))
            pytest.fail("model and oracle differ first at %s (%d vs %d bytes)" % (s.locate(i), len(s.data), len(w)))


@pytest.mark.parametrize("walk", WALKS)
def test_every_boundary_class_is_reached(models, walk):
    reached = set()
    for cid in _walk_cases(walk):
        reached |= S.classes(models(cid))
    missing = sorted(S.WALK_CLASSES[walk] - reached)
    assert not missing, "%s walk: no case reaches %s" % (walk, ", ".join(missing))


def test_placed_lengths_are_exact(built):
    """The placement solver's lengths: the 128-bit slot block at every phase of the placed tile, and the dialled
    lengths of its head, in the model of the oracle's file."""
    f, pl, _ = S.coef_case("gray_lengths:fixed")
    blocks = S.model_scans(f, pl)[0].blocks
    assert [len(b.bits) for b in blocks[:len(S.LENGTHS)]] == list(S.LENGTHS)
    assert {b.off % 32 for b in blocks[:S.TILE] if len(b.bits) == 128 and b.kind == "slot"} == set(range(32))
    assert all(b.kind == "fallback" for b in blocks[3 * S.TILE:4 * S.TILE])


COEF_IDS = [c[0] for c in S.COEF_CASES]


def _ref_scans_file(d, ncomp):
    path = os.path.join(d, "multi.txt")
    with open(path, "w") as fh:
        fh.write("".join("%d: 0 63 0 0;\n" % c for c in range(ncomp)))
    return path


@pytest.mark.parametrize("cid", COEF_IDS)
def test_oracle_matches_reference_jpegtran(built, cid):
    """jpegtran on a plain carrier of the placed planes writes the oracle's file."""
    from decode_sync_cases import encode
    from oracle import oracle as O
    if not O.ref_available() or not os.path.exists(os.path.join(O.REF_DIR, "jpegtran")):
        pytest.skip("oracle/_ref not built")
    f, pl, p = S.coef_case(cid)
    _, src, variant = next(c for c in S.COEF_CASES if c[0] == cid)
    layout, W, H, scans, _, _ = S.coef_source(src)
    carrier = encode(list(pl), layout, W, H, precision=12 if variant == "12" else 8)
    sw, scans = S.ref_switches(cid)
    with tempfile.TemporaryDirectory() as d:
        if scans == "multi":
            sw = sw + ["-scans", _ref_scans_file(d, len(pl))]
        assert O.ref_jpegtran(carrier, sw) == f


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the device writes the oracle's file; its coefficient files decode back to their planes
# ---------------------------------------------------------------------------------------------------------------------
def _device(enc, cid):
    f, pl, p = S.case(cid)
    if cid in S.PIXEL:
        return enc.encode_batch(p, S.pixel_image(cid)[None])[0]
    return enc.encode_batch_coefs(p, [a[None] for a in pl])[0]


@pytest.mark.gpu
@pytest.mark.parametrize("cid", S.ALL_CASES)
def test_device_matches_oracle(encoder, models, cid):
    f, _, _ = S.case(cid)
    got = _device(encoder, cid)
    if got != f:
        pytest.fail("device and oracle differ (%d vs %d bytes) at %s" % (len(got), len(f), S.first_difference(f, got, models(cid))))


@pytest.mark.gpu
@pytest.mark.parametrize("cid", COEF_IDS)
def test_device_coefficient_file_reads_back(encoder, cid):
    """The device's file decodes to the input planes under the serial decoder of the decode-sync suite and, where it is
    built, the reference decoder: a check that does not rest on the oracle."""
    from decode_sync_cases import serial_decode
    from oracle import oracle as O
    _, pl, _ = S.case(cid)
    got = _device(encoder, cid)
    back = serial_decode(got)
    for c, a in enumerate(pl):
        bad = np.argwhere((back[c] != a).any(-1))
        assert not len(bad), "component %d: block %s decodes differently" % (c, tuple(bad[0]))
    if O.ref_available():
        ref = O.ref_read_coefs(got)["coefs"]
        assert all((r == a).all() for r, a in zip(ref, pl))


def _batch_planes():
    """gray images of one geometry (41 x 25 blocks): the placed lengths, one of 6- and 8-bit blocks only (every block a
    slot block), one of uniform +-1023 coefficients (every block a fallback block, whatever the tables) and the restart
    placement's rule"""
    from decode_sync_cases import planes
    W, H = 41 * 8, 25 * 8
    sets = [S.placed_planes("gray_lengths"),
            S.place("gray", W, H, lambda: (lambda t, n, ph: 6 if t % 3 else 8)),
            planes("dense", "gray", W, H, 8, 5),
            S.place("gray", W, H, S.rule_restart)]
    return W, H, [[np.asarray(x) for x in s] for s in sets]


@pytest.mark.gpu
@pytest.mark.parametrize("chunk,streams", [(0, 1), (1, 1), (2, 1), (1, 2)], ids=["whole", "chunk1", "chunk2", "chunk1_streams2"])
@pytest.mark.parametrize("variant", ["opt", "fixed_restart"])
def test_device_batch_mixes_slot_and_fallback_images(built, chunk, streams, variant):
    """One batch of placed images with per-image Huffman tables (-optimize) or fixed tables and restarts: image i is the
    oracle's file of image i alone, whatever the chunking and stream count."""
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    from decode_sync_cases import params
    W, H, sets = _batch_planes()
    p = params("gray", W, H, optimize=variant == "opt", restart="3B" if variant == "fixed_restart" else None)
    e = mj.Encoder(0)
    try:
        if chunk:
            e.set_chunk_images(chunk)
        if streams > 1:
            e.set_streams(streams)
        out = e.encode_batch_coefs(p, [np.stack([s[0] for s in sets])])
    finally:
        e.close()
    for i, pl in enumerate(sets):
        want = O.oracle_encode_coefs(p, pl)
        if out[i] != want:
            pytest.fail("image %d: %s" % (i, S.first_difference(want, out[i], S.model_scans(want, pl))))
