"""jpegtran's lossless transforms (-rotate, -flip, -transpose, -transverse, -crop, -trim, -perfect, -grayscale) on
the device: the host parameter logic (b200jpeg_transform_setup) and the coefficient import's gather, from file bytes
(b200jpeg_transcode_batch_transform) and from planes (b200jpeg_encode_batch_coefs_transform).  Sources come from
tests/transform_cases.py; the expected files are the reference's own jpegtran output, recorded in
tests/golden/transform_golden.json (tools/make_golden.py --transform)."""
import json
import os
import subprocess
import sys

import pytest

import transform_cases as X
from common import GOLD, ROOT

G = json.load(open(os.path.join(GOLD, "transform_golden.json")))
CASES = {c["id"]: c for c in G["cases"]}
_cache = {}


def _src(sid):
    if sid not in _cache:
        _cache[sid] = X.source(sid)
    return _cache[sid]


def _ref_available():
    from oracle import oracle as O
    return os.path.exists(os.path.join(O.REF_DIR, "jpegtran"))


def _by_source(ids):
    out = {}
    for cid in ids:
        out.setdefault(CASES[cid]["source"], []).append(CASES[cid])
    return sorted(out.items())


MAIN = [c[0] for c in X.main_matrix()]
OTHER = [c[0] for c in X.other_cases()]


# ------------------------------------------------------------------ CPU: sources, parameters, switch parsing
def test_sources_match_recorded_files(built):
    for sid in X.source_ids():
        assert X.md5(_src(sid)[0]) == G["sources"][sid], sid


@pytest.mark.parametrize("sid,cases", _by_source(MAIN + OTHER), ids=lambda v: v if isinstance(v, str) else "")
def test_setup_reproduces_sof_and_tables(built, sid, cases):
    """params_for_transcode + b200jpeg_transform_setup give the reference output's size, components, sampling, table
    slots and (transposed) table values."""
    from mozjpeg_b200 import jpegtran as T
    info = T.parse_header(_src(sid)[0])
    for c in cases:
        p, _ = T.params_for_transcode(info, c["switches"])
        comps = [[p.comp_info[i].component_id, p.comp_info[i].h_samp_factor, p.comp_info[i].v_samp_factor, p.comp_info[i].quant_tbl_no]
                 for i in range(p.num_components)]
        assert [p.image_width, p.image_height, comps] == c["sof"], c["id"]
        assert X.tables_md5([list(p.quant_tbl[q[3]]) for q in comps]) == c["qt_md5"], c["id"]


def test_refusals_match_reference(built):
    from mozjpeg_b200 import jpegtran as T
    from mozjpeg_b200.cjpeg import UsageError
    for r in G["refusals"]:
        info = T.parse_header(_src(r["source"])[0])
        err = r["error"]
        if "Invalid crop request" in err or "not perfect" in err:
            with pytest.raises(T.TransformError, match=err.split(": ")[-1]):
                T.params_for_transcode(info, r["switches"])
        elif "Unsupported color conversion" in err:
            with pytest.raises(T.ConversionError):
                T.params_for_transcode(info, r["switches"])
        else:                                          # the reference's switch parser: usage or a named complaint
            with pytest.raises(UsageError) as e:
                T.params_for_transcode(info, r["switches"])
            if "usage" not in err:
                assert err.split(": ", 1)[1].split(" '")[0] in str(e.value), (r["switches"], str(e.value))


def test_switch_parsing(built):
    from mozjpeg_b200 import _abi as A
    from mozjpeg_b200 import jpegtran as T
    from mozjpeg_b200.cjpeg import UsageError
    info = T.parse_header(_src("227x149_420")[0])
    for sw, xf in ((["-rot", "90"], A.XFORM_ROT_90), (["-ro", "18"], None), (["-f", "h"], A.XFORM_FLIP_H), (["-flip", "v"], A.XFORM_FLIP_V),
                   (["-t"], A.XFORM_TRANSPOSE), (["-transv"], A.XFORM_TRANSVERSE), (["-tri"], A.XFORM_NONE),
                   (["-rotate", "90", "-rotate", "90"], A.XFORM_ROT_90)):
        if xf is None:
            with pytest.raises(UsageError):
                T.transcode_setup(info, sw)
            continue
        p, t, prefer = T.transcode_setup(info, sw)
        assert t.transform == xf and not prefer, sw
    assert T.transcode_setup(info, ["-perfect"])[2]                       # -perfect alone keeps prefer_smallest
    assert not T.transcode_setup(info, ["-gr"])[2]
    for sw in (["-drop", "+0+0", "x.jpg"], ["-wipe", "8x8+0+0"], ["-crop", "300x10+0+0"]):
        with pytest.raises(UsageError, match=sw[0]):
            T.transcode_setup(info, sw)
    # -progressive builds its script for the destination's component count
    p, _, _ = T.transcode_setup(info, ["-grayscale", "-progressive"])
    assert p.num_components == 1 and all(p.scan_info[k].comps_in_scan == 1 for k in range(p.num_scans))


@pytest.mark.skipif(not _ref_available(), reason="needs the reference build under oracle/_ref/")
def test_goldens_rederived_live(built):
    """the recorded outputs are what the reference's jpegtran writes for these sources today"""
    from oracle import oracle as O
    for cid in MAIN[::7] + OTHER:
        c = CASES[cid]
        out = O.ref_jpegtran(_src(c["source"])[0], c["switches"])
        assert X.md5(out) == c["md5"], cid


# ------------------------------------------------------------------ GPU: byte-identical to the reference's jpegtran
@pytest.mark.gpu
@pytest.mark.parametrize("sid,cases", _by_source(MAIN), ids=lambda v: v if isinstance(v, str) else "")
def test_main_matrix(encoder, sid, cases):
    from mozjpeg_b200 import jpegtran as T
    src = _src(sid)[0]
    for c in cases:
        out = T.transcode(encoder, [src], None, c["switches"])[0]
        assert X.md5(out) == c["md5"], c["id"]


@pytest.mark.gpu
@pytest.mark.parametrize("sid,cases", _by_source(OTHER), ids=lambda v: v if isinstance(v, str) else "")
def test_crop_grayscale_perfect_and_other_sources(encoder, sid, cases):
    from mozjpeg_b200 import jpegtran as T
    src = _src(sid)[0]
    for c in cases:
        out = T.transcode(encoder, [src], None, c["switches"])[0]
        assert X.md5(out) == c["md5"], c["id"]


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [0, 2])
def test_mixed_dqt_batch(encoder, chunk):
    """same-geometry files with different tables under -rotate 90: per-image transposed tables, equal to single runs"""
    from mozjpeg_b200 import jpegtran as T
    ids = X.mixed_ids()
    srcs = [_src(s)[0] for s in ids]
    encoder.set_chunk_images(chunk)
    try:
        out = T.transcode(encoder, srcs, None, ["-rotate", "90"])
    finally:
        encoder.set_chunk_images(0)
    assert [X.md5(o) for o in out] == [CASES[f"mixed_{s}"]["md5"] for s in ids]
    assert out == [T.transcode(encoder, [s], None, ["-rotate", "90"])[0] for s in srcs]


@pytest.mark.gpu
def test_planes_route(encoder):
    """caller planes in the source geometry: equal to the file-bytes route, and a progressive source's planes give the
    reference's jpegtran output on that progressive file"""
    from mozjpeg_b200 import jpegtran as T
    for cid in MAIN[5::97] + ["crop_64x48+5+3", "cropx7", "other1"]:
        c = CASES[cid]
        src, planes = _src(c["source"])
        out = T.transcode(encoder, [src], [pl[None] for pl in planes], c["switches"])[0]
        assert X.md5(out) == c["md5"], cid
    src, planes = _src("prog_420")
    with pytest.raises(ValueError, match="progressive"):
        T.transcode(encoder, [src], None, ["-rotate", "90"])
    for sw in (["-rotate", "90"], ["-crop", "64x48+5+3", "-transpose"]):
        out = T.transcode(encoder, [src], [pl[None] for pl in planes], sw)[0]
        assert X.md5(out) == CASES[f"prog_{'_'.join(a.lstrip('-') for a in sw)}"]["md5"], sw


@pytest.mark.gpu
@pytest.mark.skipif(not _ref_available(), reason="the CMYK / YCCK sources are the reference's TurboJPEG encodes")
def test_cmyk_ycck_from_file_bytes(encoder):
    """the CMYK / YCCK transform records of colorspace_golden.json through the file-bytes route"""
    import colorspace_cases as CC
    from mozjpeg_b200 import jpegtran as T
    recs = [t for t in json.load(open(os.path.join(GOLD, "colorspace_golden.json")))["transcode"]
            if t["switches"] in (["-rotate", "90"], ["-crop", "96x64+16+8"]) and "md5" in t]
    assert len(recs) == 4
    for t in recs:
        src = CC.tran_source(t["source"])
        assert CC.md5(src) == t["source_md5"]
        assert CC.md5(T.transcode(encoder, [src], None, t["switches"])[0]) == t["md5"], t["id"]


@pytest.mark.gpu
def test_cli(tmp_path, built):
    src = tmp_path / "in.jpg"
    src.write_bytes(_src("227x149_420")[0])
    out = tmp_path / "out.jpg"
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.jpegtran", "-rotate", "90", "-outfile", str(out), str(src)],
                       capture_output=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr.decode()
    assert X.md5(out.read_bytes()) == CASES["mixed_227x149_420"]["md5"]
    r = subprocess.run([sys.executable, "-m", "mozjpeg_b200.jpegtran", "-perfect", "-rotate", "90", "-outfile", str(tmp_path / "x.jpg"), str(src)],
                       capture_output=True, env=env, cwd=ROOT)
    assert r.returncode == 1 and b"transformation is not perfect" in r.stderr
    assert not (tmp_path / "x.jpg").exists()
