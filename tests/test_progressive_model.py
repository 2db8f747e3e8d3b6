"""The progressive decode's refinement and first-scan rules against a serial model (tests/progressive_model_cases.py):
the model on generated and recorded sources, the scan writer's round trip, constructed scans at the edges of the four
scan kinds, per-scan damage of small progressive files, pins of the model to the reference library (where its build
exists) and the device against the model.  No goldens: the CPU oracle writes every carrier from known planes."""
import json
import os

import numpy as np
import pytest

import decode_sync_cases as S
import progressive_cases as P
import progressive_model_cases as M
from common import GOLD

PROG_IDS = [c[0] for c in S.CASES if c[8] in ("prog", "script")] + [c[0] for c in S.FAMILY_CASES if c[3] == "prog"]
G = json.load(open(os.path.join(GOLD, "progressive_golden.json")))
GC = {c["id"]: c for c in G["cases"]}
RECORDED = [c[0] for c in P.CASES] + P.EXTRA_IDS
# recorded sources the device refuses although the progression check takes them (tests/test_progressive_decode.py)
RECORDED_CORRUPT = {"truncated", "corrupt", "default_restart_1"}
MODEL_MAX_BYTES = 40000                  # the serial model is plain Python
_cache = {}


def _cached(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def _recorded(sid):
    return _cached(("rec", sid), lambda: dict(P.all_sources())[sid])


def _constructed(cid):
    return _cached(("con", cid), lambda: M.constructed(cid))


def _mutants(sid):
    return _cached(("mut", sid), lambda: M.all_mutants(sid))


def _source(sid):
    return _cached(("src", sid), lambda: M.mutant_source(sid))


def _label(v):
    return "ok" if v[0] == "ok" else v[1] if v[0] == "status" else "host: " + v[1]


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("cid", PROG_IDS)
def test_model_gives_back_the_planes(built, cid):
    f, pl, _, _, _, _ = S.case_source(cid)
    for g, w in zip(M.decode(f), pl):
        np.testing.assert_array_equal(g, w)


@pytest.mark.parametrize("sid", RECORDED)
def test_model_agrees_with_the_recorded_sources(built, sid):
    """accepted sources give the reference's recorded coefficients; the sources the device refuses, the model refuses"""
    src = _recorded(sid)
    if len(src) > MODEL_MAX_BYTES:
        pytest.skip("too large for the Python model")
    try:
        verdict = P.progression(src)[0]
    except ValueError:
        verdict = "parse"
    if verdict == "sequential":
        pytest.skip("sequential source")
    v = M.verdict(src)
    if verdict in ("bad", "bogus", "parse") or sid in RECORDED_CORRUPT:
        assert v[0] != "ok", sid
    else:
        assert v[0] == "ok", _label(v)
        assert P.md5_planes(v[1]) == GC[sid]["coef_md5"]


@pytest.mark.parametrize("sid", M.MUTANT_SOURCES + ["prog_420_mixed", "script_4x1_sparse", "script12_1x4_mixed"])
def test_writer_round_trip(built, sid):
    """the tokens the model reads, written again, are the oracle's bytes"""
    f = S.case_source(sid)[0] if sid in S.CASE else _source(sid)
    assert M.rewrite(f) == f


@pytest.mark.parametrize("cid", list(M.CONSTRUCTED))
def test_constructed_verdicts(built, cid):
    f, car = _constructed(cid)
    assert M.verdict(car)[0] == "ok"
    got = _label(M.verdict(f))
    want = M.CONSTRUCTED[cid]
    if isinstance(want, str) and want.startswith("host: "):
        assert got.startswith("host: ") and want[6:] in got, got
    else:
        assert got == want


def test_every_scan_kind_reaches_both_verdicts(built):
    seen = {k: {"ok": 0, "refused": 0} for k in M.KINDS}
    for sid in M.MUTANT_SOURCES:
        for knd, _, _, m in _mutants(sid):
            seen[knd]["ok" if M.verdict(m)[0] == "ok" else "refused"] += 1
    print(seen)
    for knd, n in seen.items():
        assert n["ok"] > 0 and n["refused"] > 0, (knd, n)


def _reference_pin(f, what):
    from oracle import oracle as O
    v = M.verdict(f)
    got, warnings = O.ref_read_coefs_warn(f)
    if v[0] == "ok":
        assert got is not None, what
        for c, (g, w) in enumerate(zip(got, v[1])):
            np.testing.assert_array_equal(g, w, err_msg=f"{what} component {c}")
    elif v[0] == "status" and v[1] & -v[1] == 2 or v[0] == "host" and M.DOCUMENTED[0] in v[1]:
        pass                                       # refused where the reference decodes on silently: documented
    else:
        assert got is None or warnings > 0, (what, _label(v))


def _need_reference():
    from oracle import oracle as O
    if not O.ref_available():
        pytest.skip("no reference build")


@pytest.mark.parametrize("cid", list(M.CONSTRUCTED))
def test_reference_agrees_with_the_model_on_constructed_scans(built, cid):
    _need_reference()
    _reference_pin(_constructed(cid)[0], cid)


@pytest.mark.parametrize("sid", M.MUTANT_SOURCES)
def test_reference_agrees_with_the_model_on_damaged_files(built, sid):
    _need_reference()
    for knd, k, kd, m in _mutants(sid):
        _reference_pin(m, f"{sid} scan {k} ({knd}) {kd}")


def test_documented_refusals_are_reached(built):
    """the list of refusals the reference does not warn on is exercised: a second first scan, a value past a band"""
    assert M.DOCUMENTED[0] in M.CONSTRUCTED["second_first_scan"]
    assert M.CONSTRUCTED["refine_value_past_se"] == 2 and M.CONSTRUCTED["ac_first_value_past_se"] == 2


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def penc(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    enc.set_progressive_decode(True)
    yield enc
    enc.close()


def _pixel_route(f):
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(f)
    if info.data_precision != 8 or info.num_components not in (1, 3):
        return False
    return info.num_components == 1 or (info.h_samp_factor[0] <= 2 and info.v_samp_factor[0] <= 2 and
                                        all(info.h_samp_factor[c] == 1 and info.v_samp_factor[c] == 1 for c in (1, 2)))


def _err(fn):
    from mozjpeg_b200 import _abi as A
    with pytest.raises(A.B200JpegError) as e:
        fn()
    return e.value


def _device_against_model(enc, good, x, what):
    """read_coefficients([good, x]): image 0 the good planes, image 1 the model's planes or its refusal; the pixels of
    accepted 8-bit files in the pixel routes' layouts"""
    import recompress_cases as R
    from mozjpeg_b200 import _abi as A
    want0 = M.decode(good)
    v = M.verdict(x)
    if v[0] != "ok":
        e = _err(lambda: enc.read_coefficients([good, x]))
        words = M.STATUS_WORDS[v[1] & -v[1]] if v[0] == "status" else v[1]
        assert e.code == A.ERR_BAD_SOURCE and "image 1" in str(e) and words in str(e), (what, _label(v), str(e))
        return v
    got = enc.read_coefficients([good, x])
    for c in range(len(want0)):
        np.testing.assert_array_equal(got[c][0], want0[c], err_msg=f"{what} image 0 component {c}")
        np.testing.assert_array_equal(got[c][1], v[1][c], err_msg=f"{what} image 1 component {c}")
    if _pixel_route(x) and not P.smoothing_applies(good):
        if P.smoothing_applies(x):
            e = _err(lambda: enc.decompress([good, x]))
            assert e.code == A.ERR_UNSUPPORTED and "image 1" in str(e) and "block smoothing" in str(e), (what, str(e))
        else:
            px = enc.decompress([good, x])
            np.testing.assert_array_equal(px[0], R.decode_pixels(good, want0), err_msg=what)
            np.testing.assert_array_equal(px[1], R.decode_pixels(x, v[1]), err_msg=what)
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(M.CONSTRUCTED))
def test_constructed_scans_on_the_device(penc, cid):
    f, car = _constructed(cid)
    _device_against_model(penc, car, f, cid)
    got = penc.read_coefficients([car])
    for c, w in enumerate(M.decode(car)):
        np.testing.assert_array_equal(got[c][0], w, err_msg=f"{cid}: the carrier after the case")


@pytest.mark.gpu
@pytest.mark.parametrize("sid", M.MUTANT_SOURCES)
def test_damaged_files_on_the_device(penc, sid):
    good = _source(sid)
    for knd, k, kd, m in _mutants(sid):
        _device_against_model(penc, good, m, f"{sid} scan {k} ({knd}) {kd}")
    got = penc.read_coefficients([good])
    for c, w in enumerate(M.decode(good)):
        np.testing.assert_array_equal(got[c][0], w, err_msg=f"{sid} after its mutants")


def _mixed_files():
    """same-geometry 4:2:0 files: the standard script, a seeded script, mozjpeg's default profile, a sequential file"""
    W, H = 64, 48
    files = [S.encode(S.planes("mixed", "2x2", W, H, 8, 41), "2x2", W, H, scans="prog"),
             S.encode(S.planes("mixed", "2x2", W, H, 8, 42), "2x2", W, H, scans="script", seed=42),
             P.source(("mixed_default", W, H, 43, ["-quality", "80", "-sample", "2x2"])),
             S.encode(S.planes("mixed", "2x2", W, H, 8, 44), "2x2", W, H)]
    return files


def _ac_refine_levels(f):
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(f)
    return tuple(sum(1 for sc in info.scans[:info.num_scans] if sc.Ah and sc.Ss and sc.component_index[0] == c) for c in range(3))


def test_mixed_batch_sources_differ_in_refinement_levels(built):
    files = _mixed_files()
    assert len({_ac_refine_levels(f) for f in files[:3]}) >= 2 and len(set(_ac_refine_levels(files[0]))) > 1
    assert M.verdict(files[0])[0] == "ok" and not any(P.smoothing_applies(f) for f in files)


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 1, 3])
def test_mixed_batches_equal_single_files(penc, chunk):
    files = _mixed_files()
    penc.set_chunk_images(chunk)
    try:
        singles = [penc.read_coefficients([f]) for f in files]
        batch = penc.read_coefficients(files)
        for i, s in enumerate(singles):
            for c in range(3):
                np.testing.assert_array_equal(batch[c][i], s[c][0], err_msg=f"image {i} component {c}")
        for i, f in enumerate(files[:3]):
            for c, w in enumerate(M.decode(f)):
                np.testing.assert_array_equal(batch[c][i], w, err_msg=f"image {i} component {c} against the model")
        px = penc.decompress(files)
        for i, f in enumerate(files):
            np.testing.assert_array_equal(px[i], penc.decompress([f])[0], err_msg=f"pixels of image {i}")
    finally:
        penc.set_chunk_images(0)
