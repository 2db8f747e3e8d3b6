"""The speculative entropy decode (DESIGN §8) at its synchronisation boundaries: generated round trips, placed segment
boundaries and damaged files against a serial model.  Sources come from tests/decode_sync_cases.py; no goldens: the CPU
oracle writes every file from known coefficient planes, and entropy coding is lossless."""
import numpy as np
import pytest

import decode_sync_cases as S

SEQ_IDS = [c[0] for c in S.CASES if c[8] in ("seq", "multi")] + [c[0] for c in S.FAMILY_CASES if c[3] != "prog"]
PROG_IDS = [c[0] for c in S.CASES if c[8] in ("prog", "script")] + [c[0] for c in S.FAMILY_CASES if c[3] == "prog"]
IDS = SEQ_IDS + PROG_IDS
# 8-bit sequential cases in the layouts the pixel routes take
PIXEL_IDS = [c[0] for c in S.CASES if c[8] in ("seq", "multi") and c[5] == 8 and c[1] in S.PIXEL_LAYOUTS]
MODEL_MAX_BYTES = 40000                  # the serial model is plain Python
_cache = {}


def _src(cid):
    if cid not in _cache:
        _cache[cid] = S.case_source(cid)
    return _cache[cid]


def _batch(pls):
    """per-file plane lists -> per component (N, hib, wib, 64)"""
    return [np.stack([p[c] for p in pls]) for c in range(len(pls[0]))]


def _assert_planes(got, want, img=0, what=""):
    assert len(got) == len(want)
    for c, (g, w) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(g[img], w, err_msg=f"{what} component {c}")


@pytest.fixture(scope="module")
def penc(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    enc.set_progressive_decode(True)
    yield enc
    enc.close()


def _enc(cid, encoder, penc):
    return penc if cid in PROG_IDS else encoder


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_subsequence_constants_are_read_from_the_decoder():
    assert S.DEC_SUB_BITS % 32 == 0 and S.DEC_SUB_BITS > 0 and S.DEC_CTA > 1


@pytest.mark.parametrize("cid", IDS)
def test_generated_files_are_the_planes_for_the_reference(built, cid):
    """the premise: the oracle's files are valid encodings of their planes (where the reference build exists)"""
    from oracle import oracle as O
    if not O.ref_available():
        pytest.skip("no reference build")
    f, pl, _, _, _, _ = _src(cid)
    got = O.ref_read_coefs(f)["coefs"]
    assert len(got) == len(pl)
    for g, w in zip(got, pl):
        np.testing.assert_array_equal(g, w)


@pytest.mark.parametrize("cid", [c for c in PROG_IDS if not c.startswith("family_")])
def test_scripts_are_valid_progressions(built, cid):
    import progressive_cases as P
    from mozjpeg_b200 import jpegtran as T
    f = _src(cid)[0]
    assert P.progression(f)[0] == "ok"
    info = T.parse_source(f)
    scans = info.scans[:info.num_scans]
    if S.CASE[cid][8] == "script":                   # split bands refined on their own, and Al 13 at 12 bits
        assert any(sc.Ss > 0 and sc.Se < 63 and sc.Ah > 0 for sc in scans)
        if info.data_precision == 12:
            assert max(sc.Al for sc in scans) == 13


@pytest.mark.parametrize("cid", SEQ_IDS)
def test_serial_model_reproduces_the_planes(built, cid):
    f, pl, _, _, _, _ = _src(cid)
    if len(f) > MODEL_MAX_BYTES:
        pytest.skip("too large for the Python model")
    got = S.serial_decode(f)
    for g, w in zip(got, pl):
        np.testing.assert_array_equal(g, w)


@pytest.mark.parametrize("pid", [p for p in S.PLACED if p not in S.LARGE])
def test_placements_are_reached(built, pid):
    S.placed(pid)                                    # asserts its own placement


@pytest.mark.parametrize("sid", [m[0] for m in S.MUTANT_SOURCES])
def test_serial_model_agrees_with_the_reference_on_damaged_files(built, sid):
    """every damaged file the model accepts decodes to the model's planes in the reference too; the model refuses
    some of the damaged files and accepts others"""
    from oracle import oracle as O
    from mozjpeg_b200 import jpegtran as T
    good, pl = S.mutant_source(sid)
    info = T.parse_source(good)
    for g, w in zip(S.serial_decode(good, info), pl):
        np.testing.assert_array_equal(g, w)
    muts = S.mutants(good, 40, seed=len(sid))
    assert len(muts) == 40
    refused = 0
    for kind, m in muts:
        want = S.model(m, info)
        if want is None:
            refused += 1
            continue
        if O.ref_available():
            got = O.ref_read_coefs(m)["coefs"]
            for g, w in zip(got, want):
                np.testing.assert_array_equal(g, w, err_msg=kind)
    assert 0 < refused < len(muts)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _err(fn):
    from mozjpeg_b200 import _abi as A
    with pytest.raises(A.B200JpegError) as e:
        fn()
    return e.value


@pytest.mark.gpu
@pytest.mark.parametrize("cid", IDS)
def test_coefficients_equal_the_planes(encoder, penc, cid):
    f, pl, _, _, _, _ = _src(cid)
    _assert_planes(_enc(cid, encoder, penc).read_coefficients([f]), pl, what=cid)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c[0] for c in S.CASES])
def test_batches_equal_single_files(encoder, penc, cid):
    """three same-geometry files of different content in one call"""
    _, layout, W, H, content, prec, opt, rst, scans, seed = S.CASE[cid]
    enc = _enc(cid, encoder, penc)
    pls = [S.planes(content, layout, W, H, prec, seed + 1000 * k) for k in range(3)]
    files = [S.encode(p, layout, W, H, precision=prec, optimize=opt, restart=rst, scans=scans, seed=seed + k) for k, p in enumerate(pls)]
    got = enc.read_coefficients(files)
    for i, p in enumerate(pls):
        _assert_planes(got, p, i, f"{cid} image {i}")


@pytest.mark.gpu
@pytest.mark.parametrize("cid", IDS)
def test_transcodes_from_file_bytes_equal_transcodes_from_planes(encoder, penc, cid):
    from mozjpeg_b200 import jpegtran as T
    f, pl, _, _, _, _ = _src(cid)
    enc = _enc(cid, encoder, penc)
    for sw in ([], ["-rotate", "90"]):
        try:
            want = T.transcode(enc, [f], _batch([pl]), sw)
        except ValueError as e:
            with pytest.raises(ValueError) as e2:
                T.transcode(enc, [f], None, sw)
            assert str(e2.value) == str(e)
            continue
        assert T.transcode(enc, [f], None, sw) == want, sw


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 1, 3])
@pytest.mark.parametrize("cid", PIXEL_IDS)
def test_pixels_equal_the_numpy_decode(encoder, cid, chunk):
    import recompress_cases as R
    _, layout, W, H, content, prec, opt, rst, scans, seed = S.CASE[cid]
    n = 4 + seed % 2
    pls = [S.planes(content, layout, W, H, prec, seed + 1000 * k) for k in range(n)]
    files = [S.encode(p, layout, W, H, precision=prec, optimize=opt, restart=rst, scans=scans) for p in pls]
    encoder.set_chunk_images(chunk)
    try:
        px = encoder.decompress(files)
    finally:
        encoder.set_chunk_images(0)
    for i, (f, p) in enumerate(zip(files, pls)):
        np.testing.assert_array_equal(px[i], R.decode_pixels(f, p), err_msg=f"image {i}")


# placed cases of sequential gray files only, where the restatement predicts which CTA starts k_dec_fix must redo
GUESS_CHECKED = [p for p in S.PLACED if p not in S.LARGE and p != "periodic_420" and not p.startswith("eobrun_")]


@pytest.mark.gpu
@pytest.mark.parametrize("pid", S.PLACED)
def test_placed_boundaries(encoder, penc, pid):
    files, pls, target = S.placed(pid)             # the placement is asserted before decoding
    enc = penc if pid.startswith("eobrun_") else encoder
    got = enc.read_coefficients(files)
    rounds, redone = enc.last_decode_sync()
    t = S.segment_table(files)
    nsub = t[-1]["sub0"] + t[-1]["nsub"]
    print(f"{pid}: {nsub} subsequences, {-(-nsub // 1024)} scan tiles, {len(t)} segments; "
          f"most CTA rounds {rounds}, re-decoded {redone}")
    for i, p in enumerate(pls):
        _assert_planes(got, p, i, f"{pid} image {i}")
    if pid in GUESS_CHECKED:
        wrong = S.wrong_cta_guesses(files)
        if wrong:
            assert redone >= wrong                  # every wrongly guessed CTA start is decoded again
        else:
            assert redone == 0                      # every CTA start falls on a block start: nothing to redo
        if pid.startswith("offset_"):
            assert wrong > 0                        # the dense target's CTA starts fall inside blocks
    elif len(files) == 1 and any(s["sub0"] // S.DEC_CTA != (s["sub0"] + s["nsub"] - 1) // S.DEC_CTA for s in t):
        assert redone > 0                           # a segment crosses a CTA start: k_dec_fix had work
    if pid == "periodic_420":
        assert rounds > 100


@pytest.mark.gpu
@pytest.mark.parametrize("sid", [m[0] for m in S.MUTANT_SOURCES])
def test_damaged_files_give_the_model_planes_or_a_refusal(encoder, sid):
    import recompress_cases as R
    from mozjpeg_b200 import _abi as A
    from mozjpeg_b200 import jpegtran as T
    good, pl = S.mutant_source(sid)
    info = T.parse_source(good)
    pixels = info.data_precision == 8
    good_px = R.decode_pixels(good, pl) if pixels else None
    for k, (kind, m) in enumerate(S.mutants(good, 40, seed=len(sid))):
        want = S.model(m, info)
        what = f"{sid} mutant {k} ({kind})"
        if want is None:
            e = _err(lambda: encoder.read_coefficients([good, m]))
            assert e.code == A.ERR_BAD_SOURCE and "image 1" in str(e), (what, str(e))
            if pixels:
                e2 = _err(lambda: encoder.decompress([good, m]))
                assert e2.code == A.ERR_BAD_SOURCE and "image 1" in str(e2), (what, str(e2))
            continue
        got = encoder.read_coefficients([good, m])
        _assert_planes(got, pl, 0, what)
        _assert_planes(got, want, 1, what)
        if pixels:
            px = encoder.decompress([good, m])
            np.testing.assert_array_equal(px[0], good_px, err_msg=what)
            np.testing.assert_array_equal(px[1], R.decode_pixels(good, want), err_msg=what)
    _assert_planes(encoder.read_coefficients([good]), pl, 0, f"{sid} after its mutants")
