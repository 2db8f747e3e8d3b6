"""Device decode of progressive Huffman JPEG files (b200jpeg_encoder_set_progressive_decode) through every decode entry
point.  Sources come from tests/progressive_cases.py; the reference's coefficients, jpegtran outputs and pixels for them
are in tests/golden/progressive_golden.json (tools/make_golden.py --progressive).  The GPU tests use an encoder of their
own with progressive decode on, so the session encoder keeps the default (off)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import progressive_cases as P
from common import GOLD, ROOT

G = json.load(open(os.path.join(GOLD, "progressive_golden.json")))
GC = {c["id"]: c for c in G["cases"]}
IDS = [c[0] for c in P.CASES] + P.EXTRA_IDS
# decoded with warnings by the reference (its data runs out or holds invalid codes); the device refuses them.
# default_restart_1: the default profile's scan search writes one restart interval (the first scan's DRI) for scans
# whose data restarts at another interval, so a decoder finds RSTn markers where it does not expect them
CORRUPT = {"truncated", "corrupt", "default_restart_1"}
_cache = {}


def _src(sid):
    if sid not in _cache:
        _cache.update(P.all_sources())
    return _cache[sid]


def _verdict(sid):
    try:
        return P.progression(_src(sid))[0]
    except ValueError:
        return "parse"


def _refused(sid):
    return _verdict(sid) in ("bad", "bogus", "parse") or sid in CORRUPT


def _pixel_route(sid):
    """None when the pixel routes take the source, else the words of their refusal"""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_source(_src(sid))
    if info.data_precision != 8:
        return "12-bit"
    if info.num_components not in (1, 3):
        return "4-component"
    if info.num_components == 3 and (info.h_samp_factor[0] > 2 or info.v_samp_factor[0] > 2 or
                                     any(info.h_samp_factor[c] != 1 or info.v_samp_factor[c] != 1 for c in (1, 2))):
        return "sampling layout"
    if P.smoothing_applies(_src(sid)):
        return "block smoothing"
    return None


@pytest.fixture(scope="module")
def penc(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    enc.set_progressive_decode(True)
    yield enc
    enc.close()


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("sid", IDS)
def test_sources_match_recorded_files(built, sid):
    assert P.md5(_src(sid)) == GC[sid]["src_md5"]


@pytest.mark.parametrize("sid", IDS)
def test_progression_check_agrees_with_the_reference(built, sid):
    """what the restated checks accept, the reference decodes without error; JERR_BAD_PROGRESSION files it refuses"""
    v = _verdict(sid)
    if v in ("ok", "sequential", "bogus"):
        assert "coef_md5" in GC[sid], GC[sid]
    else:
        assert "coef_error" in GC[sid]


@pytest.mark.parametrize("sid", IDS)
def test_smoothing_restatement_agrees_with_the_reference(built, sid):
    """smoothing_applies against the recorded verdict of the reference library (pixels with do_block_smoothing on and
    off differ), for every source the progression check accepts and the reference decodes to pixels"""
    if _verdict(sid) not in ("ok", "sequential") or GC[sid]["ref_smooths"] is None:
        pytest.skip("not decoded to pixels by the reference, or refused by the progression check")
    assert P.smoothing_applies(_src(sid)) == GC[sid]["ref_smooths"]


# ---------------------------------------------------------------------------------------------------------------- GPU
def _err(fn):
    from mozjpeg_b200 import _abi as A
    with pytest.raises(A.B200JpegError) as e:
        fn()
    return e.value


@pytest.mark.gpu
@pytest.mark.parametrize("sid", IDS)
def test_coefficients_equal_the_reference(penc, sid):
    from mozjpeg_b200 import _abi as A
    src = _src(sid)
    if _verdict(sid) == "parse":                      # the header parser refuses it (a table the scan needs is missing)
        with pytest.raises((ValueError, A.B200JpegError)):
            penc.read_coefficients([src])
        return
    if _refused(sid):
        e = _err(lambda: penc.read_coefficients([src]))
        assert e.code == A.ERR_BAD_SOURCE and "image 0" in str(e)
        return
    got = penc.read_coefficients([src])
    assert P.md5_planes([p[0] for p in got]) == GC[sid]["coef_md5"]


@pytest.mark.gpu
@pytest.mark.parametrize("sid", [s for s in IDS if s not in CORRUPT])
def test_transcodes_equal_the_reference_jpegtran(penc, sid):
    from mozjpeg_b200 import jpegtran as T
    if _refused(sid):
        pytest.skip("refused source")
    for sw in G["jpegtran_switches"]:
        want = GC[sid]["jpegtran"][" ".join(sw)]
        if want is None:
            continue
        try:
            out = T.transcode(penc, [_src(sid)], None, sw)[0]
        except ValueError as e:                           # a crop past a small image: crop extension is not on the device path
            if sw[0] == "-crop" and "crop extension" in str(e):
                continue
            raise
        assert P.md5(out) == want, (sid, sw)


@pytest.mark.gpu
@pytest.mark.parametrize("sid", [s for s in IDS if s not in CORRUPT])
def test_pixels_equal_the_reference(penc, sid):
    from mozjpeg_b200 import _abi as A
    if _refused(sid):
        pytest.skip("refused source")
    why = _pixel_route(sid)
    if why:
        e = _err(lambda: penc.decompress([_src(sid)]))
        assert e.code == A.ERR_UNSUPPORTED and "image 0" in str(e) and why.split()[0] in str(e), str(e)
        if why == "block smoothing":
            assert GC[sid]["ref_smooths"] is True           # refused only where the reference does smooth
        return
    px = penc.decompress([_src(sid)])[0]
    assert P.md5(px) == GC[sid]["pix_md5"]


@pytest.mark.gpu
@pytest.mark.parametrize("sid", ["default_q75", "sample_420", "gray", "restart_1"])
def test_recompression_equals_encoding_the_decoded_pixels(penc, sid):
    import mozjpeg_b200 as mj
    src = _src(sid)
    p = mj.params_for_jpeg_input(["-quality", "75"], src)
    px = penc.decompress([src])
    assert penc.recompress(p, [src])[0] == penc.encode_batch(mj.params_for_jpeg_input(["-quality", "75"], src), px)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("sw", [[], ["-progressive", "-revert"], ["-quality", "95", "-restart", "2"], ["-sample", "1x1", "-dc-scan-opt", "2"]])
def test_device_encoder_outputs_round_trip(penc, sw):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    imgs = np.stack([O.synth_image(s, 96, 64) for s in (31, 32)])
    p = mj.params_from_switches(sw, 96, 64)
    files = penc.encode_batch(p, imgs)
    planes = penc.read_coefficients(files)
    p.trellis_quant = 0                                   # the coefficients are quantized already (jpeg_copy_critical_parameters)
    assert penc.encode_batch_coefs(p, planes) == files


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 2])
def test_mixed_sequential_and_progressive_batches(penc, chunk):
    import mozjpeg_b200 as mj
    from oracle import oracle as O
    files = []
    for k, sw in enumerate([["-revert"], [], ["-progressive", "-revert", "-restart", "1"], ["-revert", "-restart", "2"], ["-quality", "40"]]):
        p = mj.params_from_switches(sw, 80, 48)
        files.append(O.oracle_encode(p, O.synth_image(40 + k, 80, 48)).jpeg)
    penc.set_chunk_images(chunk)
    try:
        singles = [penc.read_coefficients([f]) for f in files]
        batch = penc.read_coefficients(files)
        for i, s in enumerate(singles):
            for c in range(3):
                np.testing.assert_array_equal(batch[c][i], s[c][0])
        px = penc.decompress(files)
        for i, f in enumerate(files):
            np.testing.assert_array_equal(px[i], penc.decompress([f])[0])
        p = mj.params_for_jpeg_input(["-quality", "70"], files[0])
        assert penc.recompress(p, files) == [penc.recompress(p, [f])[0] for f in files]
    finally:
        penc.set_chunk_images(0)


@pytest.mark.gpu
def test_refusals_name_the_image_and_the_encoder_recovers(penc):
    from mozjpeg_b200 import _abi as A
    good = _src("default_q75")
    for sid, code, words in (("swap_scans", A.ERR_BAD_SOURCE, "bogus progression"), ("wrong_ah", A.ERR_BAD_SOURCE, "bogus progression"),
                             ("ac_before_dc", A.ERR_BAD_SOURCE, "before its DC scan"), ("two_component_ac", A.ERR_BAD_SOURCE, "AC Huffman table"),
                             ("two_component_ac_tables", A.ERR_BAD_SOURCE, "scan 3: bad progression parameters Ss=1 Se=63 Ah=0 Al=1"),
                             ("al_14", A.ERR_BAD_SOURCE, "scan 0: bad progression parameters Ss=0 Se=0 Ah=0 Al=14"),
                             ("truncated", A.ERR_BAD_SOURCE, "corrupt entropy-coded data")):
        e = _err(lambda: penc.read_coefficients([good, _src(sid)]))
        assert e.code == code and "image 1" in str(e) and words in str(e), (sid, str(e))
    e = _err(lambda: penc.decompress([good, good, _src("drop_to_dc_only")]))
    assert e.code == A.ERR_UNSUPPORTED and "image 2" in str(e) and "block smoothing" in str(e)
    got = penc.read_coefficients([good])
    assert P.md5_planes([p[0] for p in got]) == GC["default_q75"]["coef_md5"]


@pytest.mark.gpu
def test_switch_off_keeps_todays_refusals(encoder):
    from mozjpeg_b200 import _abi as A, jpegtran as T
    src = _src("default_q75")
    e = _err(lambda: encoder.read_coefficients([src]))
    assert e.code == A.ERR_UNSUPPORTED and "progressive (SOF2) source: the device decode takes sequential files" in str(e)
    e = _err(lambda: encoder.decompress([src]))
    assert e.code == A.ERR_UNSUPPORTED and "progressive (SOF2) source: only sequential files are decoded to pixels" in str(e)
    with pytest.raises(ValueError):
        T.transcode(encoder, [src], None, [])


@pytest.mark.gpu
def test_command_lines_read_progressive_files(tmp_path):
    sid = "default_q75"
    src = tmp_path / "in.jpg"
    src.write_bytes(_src(sid))
    out = tmp_path / "t.jpg"
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.jpegtran", "-rotate", "90", "-outfile", str(out), str(src)], capture_output=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    assert P.md5(out.read_bytes()) == GC[sid]["jpegtran"]["-rotate 90"]
    ppm = tmp_path / "o.ppm"
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.djpeg", "-outfile", str(ppm), str(src)], capture_output=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    body = ppm.read_bytes()
    assert P.md5(np.frombuffer(body[-200 * 136 * 3:], np.uint8)) == GC[sid]["pix_md5"]
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.cjpeg", "-quality", "60", "-outfile", str(tmp_path / "c.jpg"), str(src)], capture_output=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "c.jpg").read_bytes()[:2] == b"\xff\xd8"
