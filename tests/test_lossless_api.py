"""Lossless JPEG (SOF3) through the project's drop-in boundary: the libjpeg API (jpeg_start_compress, jpeg_write_scanlines,
jpeg12_ / jpeg16_write_scanlines, jpeg_finish_compress) and the TurboJPEG API on top of it, as an unmodified application
reaches them with the interposer preloaded or the standalone libjpeg.so.62 linked.  Every output is compared with what
the reference library writes for the same calls."""
import ctypes as C
import hashlib
import json
import os
import shutil
import subprocess
import sys
import zlib

import numpy as np
import pytest

from common import GOLD, ROOT

REF = os.path.join(ROOT, "oracle", "_ref")
SHIM = os.path.join(ROOT, "integration", "_build", "libjpeg_b200shim.so")
CJPEG = os.path.join(REF, "cjpeg")
TJBENCH = os.path.join(REF, "tjbench")
REF_LIB = os.path.join(REF, "libjpeg_ref.so")
STD_LIB = os.path.join(ROOT, "integration", "_build", "libjpeg.so.62")
STD_CJPEG = os.path.join(ROOT, "integration", "_build", "cjpeg_b200")
PPM = os.path.join(GOLD, "testorig.ppm")
REFLL = os.path.join(ROOT, "build", "librefll.so")

need_shim = pytest.mark.skipif(not (os.path.exists(SHIM) and os.path.exists(CJPEG)),
                               reason="shim / reference cjpeg not built (needs the reference at build time)")
need_std = pytest.mark.skipif(not (os.path.exists(STD_LIB) and os.path.exists(STD_CJPEG) and os.path.exists(CJPEG)),
                              reason="standalone libjpeg.so.62 not built (needs the reference at build time)")
need_refll = pytest.mark.skipif(not (os.path.exists(SHIM) and os.path.exists(REFLL)),
                                reason="tests/refll.c driver not built (needs the reference at build time)")
DEVICE = {"LD_PRELOAD": SHIM, "B200_SHIM_REQUIRE": "1", "B200_SHIM_VERBOSE": "1"}


def write_pnm(path, a, maxval):
    """a: (h, w) or (h, w, 3) samples; written as binary PGM / PPM, 16-bit big-endian samples above maxval 255"""
    h, w = a.shape[:2]
    magic = b"P6" if a.ndim == 3 else b"P5"
    data = a.astype(">u2").tobytes() if maxval > 255 else a.astype(np.uint8).tobytes()
    with open(path, "wb") as f:
        f.write(magic + b"\n%d %d\n%d\n" % (w, h, maxval) + data)


def sample_image(seed, h, w, nc, prec):
    rng = np.random.default_rng(seed)
    top = (1 << prec) - 1
    yy, xx = np.mgrid[0:h, 0:w]
    base = (xx * 5 + yy * 3)[..., None] * (top // 255 + 1) + np.arange(nc) * 29
    a = (base + rng.integers(0, max(2, top // 50), size=(h, w, nc))) % (top + 1)
    return a[..., 0] if nc == 1 else a


# ---------------------------------------------------------------- CPU
@need_std
def test_standalone_libjpeg_exports_jpeg16_write_scanlines():
    """jpeg16_write_scanlines is the reference's own, with its version: 16-bit rows reach the device through the main
    controller the shim installs, so the entry point is not renamed."""
    out = subprocess.check_output(["nm", "-D", "--defined-only", STD_LIB], text=True)
    have = {}
    for ln in out.splitlines():
        f = ln.split()
        if len(f) == 3 and f[1] == "T":
            name, _, ver = f[2].partition("@@")
            have[name] = ver
    assert have.get("jpeg16_write_scanlines") == "LIBJPEG_6.2"
    assert not [n for n in have if n.startswith("b200ref_")]
    local = subprocess.check_output(["nm", "--defined-only", STD_LIB], text=True).split()
    assert "b200ref_jpeg16_write_scanlines" not in local and "b200ref_jpeg12_write_scanlines" in local


@need_std
@pytest.mark.parametrize("prec", [8, 16])
def test_standalone_lossless_without_a_device_is_the_reference(prec, tmp_path):
    """With the device path unavailable, the standalone library hands lossless objects to the reference code it carries,
    at 8 and 16 bits."""
    if prec == 8:
        src, sw = PPM, ["-revert", "-lossless", "4,1", "-restart", "2"]
    else:
        src, sw = str(tmp_path / "in16.ppm"), ["-revert", "-precision", "16", "-lossless", "6,3"]
        write_pnm(src, sample_image(16, 31, 45, 3, 16), 65535)
    a = subprocess.run([STD_CJPEG, *sw, src], env=dict(os.environ, MOZ_B200_FORCE_CPU="1", B200_SHIM_VERBOSE="1"), capture_output=True, timeout=300)
    b = subprocess.run([CJPEG, *sw, src], capture_output=True, timeout=300)
    assert a.returncode == 0 and b.returncode == 0, a.stderr + b.stderr
    assert b"reference path" in a.stderr
    assert a.stdout == b.stdout and a.stdout[:2] == b"\xff\xd8" and b"\xff\xc3" in a.stdout


def test_total_passes_of_lossless_blocks():
    """The progress monitor's pass count for lossless objects: two passes per scan (optimal tables are forced)."""
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import _abi as A
    lib = A.load()
    p = mj.params_from_switches(["-revert", "-lossless", "3"], 32, 16, 3)
    assert lib.b200jpeg_total_passes(C.byref(p)) == 2
    p = mj.params_from_switches(["-revert", "-precision", "16", "-lossless", "7,2"], 32, 16, 1)
    assert lib.b200jpeg_total_passes(C.byref(p)) == 2
    for script in ([((0, 1, 2), 1, 0)], [((0, 2), 6, 0), ((1,), 5, 4)], [((0,), 1, 0), ((1,), 2, 0), ((2,), 3, 1)]):
        q = mj.params_from_switches(["-revert"], 32, 16, 3)
        q.num_scans = len(script)
        for i, (comps, ss, al) in enumerate(script):
            e = q.scan_info[i]
            e.comps_in_scan = len(comps)
            for k in range(4):
                e.component_index[k] = comps[k] if k < len(comps) else 0
            e.Ss, e.Se, e.Ah, e.Al = ss, 0, 0, al
        q.optimize_coding = 0
        assert lib.b200jpeg_validate(C.byref(q)) == 0
        assert lib.b200jpeg_total_passes(C.byref(q)) == 2 * len(script)


# ---------------------------------------------------------------- GPU
# Runs test_lossless.py's cases through tests/refll.c (cjpeg's call sequence on the libjpeg API) in a process with the
# interposer in front of the reference library, and prints each case's md5 or the reference's error text.
_CHILD = r"""
import hashlib, json, sys, zlib
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import test_lossless as L
out = []
for c in json.loads(sys.stdin.read()):
    sw, cs, nc, prec, (h, w), kind, script = c
    script = [(tuple(comps), ss, al) for comps, ss, al in script] if script else None
    pix = L.image(zlib.crc32(L._id((sw, cs, nc, prec, (h, w), kind, script)).encode()), h, w, nc, prec, kind)
    try:
        out.append(hashlib.md5(L.ref_encode(pix, sw, cs, script)).hexdigest())
    except RuntimeError as e:
        out.append("error: " + str(e))
print(json.dumps(out))
"""


def run_cases_under_interposer(cases, env_extra):
    env = dict(os.environ, LD_PRELOAD=SHIM + ":" + REF_LIB, B200_SHIM_VERBOSE="1", **env_extra)
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, os.path.join(ROOT, "tests")], input=json.dumps(cases), env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1]), r.stderr


@need_refll
@pytest.mark.gpu
def test_every_golden_case_through_the_libjpeg_api():
    import test_lossless as L
    got, err = run_cases_under_interposer(L.CASES, {"B200_SHIM_REQUIRE": "1"})
    want = [L.GOLDEN[L._id(c)] for c in L.CASES]
    bad = [L._id(c) for c, g, w in zip(L.CASES, got, want) if g != w]
    assert not bad, bad
    assert err.count("b200 shim: device path") == len(L.CASES) and "reference path" not in err, err[-4000:]
    assert err.count("device path (lossless") == len(L.CASES) - 1          # the progressive script over -lossless is lossy


@need_refll
@pytest.mark.gpu
def test_fall_throughs_keep_the_reference_result():
    """Parameter sets the device path does not take reach the reference, with its error text or its bytes: lossless with
    the trellis on, a point transform at the data precision, lossless beside the scan search's script (SOF2 headers)."""
    import test_lossless as L
    from mozjpeg_b200 import _abi as A
    cases = [(["-baseline", "-lossless", "2"], A.CS_RGB, 3, 8, (16, 16), "smooth", None),
             (["-revert"], A.CS_RGB, 3, 8, (16, 16), "smooth", [((0, 1, 2), 1, 8)]),
             (["-notrellis", "-lossless", "1"], A.CS_RGB, 3, 8, (16, 16), "smooth", None)]
    got, err = run_cases_under_interposer(cases, {})
    want = []
    for sw, cs, nc, prec, (h, w), kind, script in cases:
        pix = L.image(zlib.crc32(L._id((sw, cs, nc, prec, (h, w), kind, script)).encode()), h, w, nc, prec, kind)
        try:
            want.append(hashlib.md5(L.ref_encode(pix, sw, cs, script)).hexdigest())
        except RuntimeError as e:
            want.append("error: " + str(e))
    assert got == want
    assert [g.startswith("error") for g in got] == [True, True, False]
    assert err.count("b200 shim: reference path") == 3 and "b200 shim: device path" not in err, err


def _cjpeg_inputs(tmp_path):
    a12 = sample_image(12, 53, 71, 3, 12)
    write_pnm(tmp_path / "in12.ppm", a12, 4095)
    write_pnm(tmp_path / "in12.pgm", a12[..., 1], 4095)
    a16 = sample_image(16, 47, 66, 3, 16)
    write_pnm(tmp_path / "in16.ppm", a16, 65535)
    write_pnm(tmp_path / "in16.pgm", a16[..., 2], 65535)
    return {"ppm8": PPM, "ppm12": str(tmp_path / "in12.ppm"), "pgm12": str(tmp_path / "in12.pgm"),
            "ppm16": str(tmp_path / "in16.ppm"), "pgm16": str(tmp_path / "in16.pgm")}


CJPEG_SETS = [("ppm8", ["-revert", "-lossless", "1"]), ("ppm8", ["-revert", "-lossless", "5,2", "-restart", "3"]),
              ("ppm8", ["-baseline", "-notrellis", "-lossless", "7,1"]), ("ppm8", ["-revert", "-lossless", "4", "-restart", "227B"]),
              ("ppm12", ["-revert", "-precision", "12", "-lossless", "6,3"]), ("pgm12", ["-revert", "-precision", "12", "-lossless", "2", "-restart", "1"]),
              ("ppm16", ["-revert", "-precision", "16", "-lossless", "4,5", "-restart", "2"]), ("pgm16", ["-revert", "-precision", "16", "-lossless", "1"]),
              ("ppm16", ["-revert", "-precision", "16", "-lossless", "7", "-grayscale"])]


@need_shim
@need_std
@pytest.mark.gpu
@pytest.mark.parametrize("src,sw", CJPEG_SETS, ids=lambda v: v if isinstance(v, str) else "_".join(x.lstrip("-") for x in v))
def test_reference_cjpeg_lossless_runs_on_the_device(src, sw, tmp_path):
    """The reference's cjpeg binary under the interposer, and its front end on the standalone library, write the
    reference's bytes with the encode on the device."""
    path = _cjpeg_inputs(tmp_path)[src]
    plain = subprocess.run([CJPEG, *sw, path], capture_output=True, timeout=300)
    assert plain.returncode == 0 and b"\xff\xc3" in plain.stdout
    pre = subprocess.run([CJPEG, *sw, path], env=dict(os.environ, **DEVICE), capture_output=True, timeout=300)
    std = subprocess.run([STD_CJPEG, *sw, path], env=dict(os.environ, B200_SHIM_REQUIRE="1", B200_SHIM_VERBOSE="1"), capture_output=True, timeout=300)
    for r in (pre, std):
        assert r.returncode == 0, r.stderr
        assert b"device path (lossless" in r.stderr, r.stderr
        assert r.stdout == plain.stdout


# the pixel formats test_libjpeg_shim.py's TurboJPEG test uses (None: tjbench's default, BGR)
TJ_FORMATS = [None, "-rgb", "-rgbx", "-bgrx", "-xbgr", "-xrgb"]


@pytest.mark.skipif(not (os.path.exists(SHIM) and os.path.exists(TJBENCH)), reason="shim / reference tjbench not built")
@pytest.mark.gpu
@pytest.mark.parametrize("prec,psv,extra", [(8, "4", []), (12, "6", ["-restart", "1"]), (16, "7", [])], ids=["p8", "p12", "p16"])
@pytest.mark.parametrize("fmt", TJ_FORMATS, ids=lambda f: (f or "-bgr").lstrip("-"))
def test_tjbench_lossless_runs_on_the_device(prec, psv, extra, fmt, tmp_path):
    """tjbench -lossless (tj3Compress8/12/16 with TJPARAM_LOSSLESS; the quality argument is the predictor) writes the
    same file with the interposer as without it."""
    outs = []
    for name, env_extra in (("dev", DEVICE), ("ref", {})):
        d = tmp_path / name
        d.mkdir()
        if prec == 8:
            shutil.copyfile(PPM, d / "img.ppm")
        else:
            write_pnm(d / "img.ppm", sample_image(prec, 61, 83, 3, prec), (1 << prec) - 1)
        r = subprocess.run([TJBENCH, "img.ppm", psv, *([fmt] if fmt else []), "-precision", str(prec), "-lossless", "-quiet", "-benchtime", "0.01",
                            "-warmup", "0", "-componly", *extra], cwd=d, env=dict(os.environ, **env_extra), capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr + r.stdout
        if name == "dev":
            assert "device path (lossless" in r.stderr and "reference path" not in r.stderr, r.stderr
        jpgs = sorted(f for f in os.listdir(d) if f.endswith(".jpg"))
        assert len(jpgs) == 1, os.listdir(d)
        outs.append((d / jpgs[0]).read_bytes())
    assert outs[0] == outs[1] and b"\xff\xc3" in outs[0]


@pytest.mark.skipif(not (os.path.exists(SHIM) and os.path.exists(os.path.join(REF, "libturbojpeg_ref.so"))), reason="shim / reference not built")
@pytest.mark.gpu
def test_c_application_under_the_interposer(tmp_path):
    """tests/refllapi.c prints the same thing with the interposer preloaded as without it: the files of tj3Compress8/12/16
    and of libjpeg-API objects, every progress-monitor call, and the object's fields after jpeg_start_compress."""
    exe = tmp_path / "refllapi"
    subprocess.check_call(["gcc", "-O2", "-w", "-I" + os.path.join(REF, "cfg"), "-I" + os.path.join(REF, "inc"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "refllapi.c"), "-L" + REF, "-lturbojpeg_ref", "-ljpeg_ref", "-Wl,-rpath," + REF])
    dev = subprocess.run([str(exe)], env=dict(os.environ, **DEVICE), capture_output=True, text=True, timeout=300)
    ref = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert dev.returncode == 0 and ref.returncode == 0, dev.stderr + ref.stderr
    assert dev.stdout == ref.stdout
    assert "error" not in ref.stdout and ref.stdout.count("progress 1 ") > 100
    # 12 TurboJPEG calls and 9 libjpeg objects, all on the device; the progressive script over jpeg_enable_lossless is lossy
    assert dev.stderr.count("b200 shim: device path") == 21 and dev.stderr.count("device path (lossless") == 20, dev.stderr
    assert ref.stdout.splitlines()[-2].split() == ["lossless", "0"]
