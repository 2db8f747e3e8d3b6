#!/usr/bin/env python3
"""Generate tests/golden/golden.json from the UNMODIFIED reference.

Runs only where /root/reference exists (oracle/_ref built by oracle/Makefile).
For every case it records the md5 and size of what the reference encoder
produces; the tests then hold the CPU oracle and the CUDA path to those
numbers on machines where the reference is absent.

Inputs are either the reference's own test image (testimages/testorig.ppm,
copied to tests/golden/ as a data fixture) or synthetic images generated from
a seed by oracle.synth_image (SURVEY 8d).
"""
import hashlib, json, os, shutil, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from oracle import oracle as O
import mozjpeg_b200 as cjpeg

REF = "/root/reference"
GOLD = os.path.join(ROOT, "tests", "golden")

SWITCH_SETS = [
    ["-revert", "-dct", "int"],                       # == testimages/testimgint.jpg, CMakeLists.txt:1391 (config 1)
    ["-revert", "-optimize"],
    ["-revert", "-progressive"],
    ["-revert", "-quality", "90", "-sample", "2x2"],
    ["-revert", "-sample", "1x1"],                    # ~ 444-islow family
    ["-revert", "-sample", "2x1", "-optimize"],       # ~ 422-*-opt family
    ["-revert", "-sample", "1x2"],                    # ~ 440-islow
    ["-revert", "-grayscale"],                        # ~ gray-islow
    ["-revert", "-grayscale", "-progressive"],
    ["-baseline", "-quality", "75"],                  # config 2 semantics (4:2:0 is the default)
    ["-baseline", "-quality", "75", "-sample", "2x2"],
    ["-baseline", "-quality", "50", "-sample", "2x2"],
    ["-baseline", "-quality", "90", "-sample", "2x2"],
    ["-baseline", "-quality", "75", "-sample", "1x1"],
    ["-baseline", "-quality", "85"],
    ["-baseline", "-quality", "95"],
    ["-baseline", "-quality", "100"],
    ["-baseline", "-quality", "20"],
    ["-baseline", "-notrellis", "-quality", "75"],
    ["-baseline", "-notrellis-dc", "-quality", "75"],
    ["-baseline", "-noovershoot", "-quality", "75"],
    ["-baseline", "-grayscale", "-quality", "75"],
    ["-baseline", "-quant-table", "2", "-quality", "80"],
    ["-baseline", "-lambda1", "12.0", "-lambda2", "13.0", "-quality", "75"],
    ["-fastcrush", "-quality", "75"],                 # config 3 semantics
    ["-fastcrush", "-quality", "75", "-sample", "2x2"],
    ["-fastcrush", "-quality", "50", "-sample", "2x2"],
    ["-fastcrush", "-quality", "90", "-sample", "2x2"],
    ["-fastcrush", "-quality", "92"],
    ["-fastcrush", "-grayscale", "-quality", "75"],
    ["-fastcrush", "-notrellis", "-quality", "75"],
    ["-baseline", "-quality", "75", "-restart", "1"],
    ["-fastcrush", "-quality", "75", "-restart", "2"],
    ["-revert", "-restart", "3B"],
    # the library default: 64-scan (23 for gray) search, jcparam.c:733-852 + jcmaster.c:773-962
    ["-quality", "75"],
    ["-quality", "90"],
    ["-quality", "50", "-sample", "2x2"],
    ["-grayscale", "-quality", "75"],
    ["-quality", "75", "-restart", "1"],
    ["-quality", "85", "-notrellis"],
    # JDCT_FLOAT (jfdctflt.c; this reference build is the "no-fp-contract" flavour of CMakeLists.txt:965-1024)
    ["-dct", "float", "-baseline", "-quality", "75"],
    ["-dct", "float", "-quality", "75", "-fastcrush"],
    ["-dct", "float", "-baseline", "-notrellis", "-quality", "90", "-sample", "1x1"],
    ["-dct", "float", "-baseline", "-quality", "50", "-grayscale"],
    ["-dct", "float", "-quality", "75"],
    # JDCT_IFAST (jfdctfst.c, scaled divisors + reciprocal quantizer)
    ["-dct", "fast", "-baseline", "-quality", "75"],
    ["-dct", "fast", "-fastcrush", "-quality", "40"],
    ["-dct", "fast", "-baseline", "-notrellis", "-quality", "95", "-sample", "1x1"],
    ["-dct", "fast", "-baseline", "-quality", "100", "-grayscale"],
    ["-dct", "fast", "-quality", "75"],
]
# input smoothing (jcsample.c:298-455, context-row mode of jcprepct.c) and sampling layouts that go through
# int_downsample (jcsample.c:151-190); the refshim driver hands these to the reference's cjpeg binary
SWITCH_SETS_EXTRA = [
    ["-revert", "-smooth", "10"],
    ["-baseline", "-quality", "75", "-smooth", "30"],
    ["-quality", "75", "-smooth", "100", "-sample", "1x1"],
    ["-baseline", "-quality", "80", "-smooth", "50", "-sample", "2x1"],
    ["-revert", "-smooth", "20", "-sample", "3x2"],
    ["-baseline", "-grayscale", "-smooth", "15", "-quality", "60"],
    ["-fastcrush", "-smooth", "5", "-sample", "2x2,1x1,2x2"],
    ["-dct", "float", "-baseline", "-quality", "75", "-smooth", "40"],
    # vertical-gradient weight in the DC trellis (jcdctmgr.c:1069-1086): acts on components with v_samp_factor > 1
    ["-baseline", "-quality", "75", "-trellis-dc-ver-weight", "1.0"],
    ["-quality", "85", "-trellis-dc-ver-weight", "0.5", "-sample", "2x2"],
    ["-fastcrush", "-quality", "60", "-trellis-dc-ver-weight", "2.5", "-sample", "1x2"],
    # cjpeg's tuning presets (cjpeg.c:678-704): base table index + lambda scales; -tune-psnr has lambda_log_scale2 = 0,
    # i.e. the constant-lambda branch of quantize_trellis (jcdctmgr.c:1031-1035)
    ["-tune-psnr"], ["-tune-ssim"], ["-tune-ms-ssim"], ["-tune-hvs-psnr"],
    ["-tune-psnr", "-quality", "85", "-baseline"],
    ["-baseline", "-lambda1", "10.5", "-lambda2", "0", "-quality", "70"],
    ["-revert", "-sample", "3x2"],
    ["-baseline", "-quality", "75", "-sample", "4x2"],
    ["-quality", "75", "-sample", "3x1"],
    ["-baseline", "-quality", "80", "-sample", "2x2,1x1,2x2"],
    ["-baseline", "-sample", "4x1,1x1,2x1", "-quality", "60"],
    # fast / float DCT on sampling layouts outside the tiled kernel's (the one-thread-per-block forward kernel)
    ["-baseline", "-quality", "75", "-sample", "3x1", "-dct", "fast"],
    ["-quality", "80", "-sample", "4x2", "-dct", "float"],
    ["-fastcrush", "-quality", "75", "-sample", "2x2,1x1,2x2", "-dct", "fast"],
    ["-baseline", "-quality", "75", "-sample", "3x2", "-dct", "float", "-smooth", "20"],
    ["-baseline", "-quality", "75", "-rgb", "-dct", "float"],
]
# switches that name files (rdswitch.c read_quant_tables / set_quant_slots / read_scan_script); "@GOLD/" = tests/golden/
SWITCH_SETS_FILES = [
    ["-qtables", "@GOLD/qtables_a.txt", "-quality", "75"],
    ["-qtables", "@GOLD/qtables_a.txt", "-baseline"],
    ["-quality", "60,90", "-qtables", "@GOLD/qtables_a.txt", "-qslots", "1,0,0"],
    ["-quality", "70,80", "-qslots", "1,0,1"],
    ["-scans", "@GOLD/scans_a.txt", "-quality", "75"],                       # successive approximation, band splits
    ["-scans", "@GOLD/scans_b.txt", "-quality", "80"],                       # sequential, two scans
    ["-scans", "@GOLD/scans_c.txt"],
    ["-revert", "-scans", "@GOLD/scans_a.txt"],
    ["-revert", "-scans", "@GOLD/scans_b.txt", "-optimize"],
    ["-scans", "@GOLD/scans_c.txt", "-restart", "1", "-sample", "2x1"],
]
# through the reference's cjpeg binary only (our refshim driver does not parse these switches)
CJPEG_ONLY = [
    ["-revert", "-dct", "float"],
    ["-revert", "-dct", "float", "-optimize", "-progressive"],
    ["-revert", "-dct", "fast"],
    ["-quality", "75", "-dc-scan-opt", "2"],
    ["-quality", "60", "-dc-scan-opt", "1"],
    ["-quality", "85", "-dc-scan-opt", "0"],
]
# 12-bit precision (config 5 semantics and relatives): the reference can only run these with the trellis and the
# deringing off (SURVEY F5); optimal Huffman tables are forced (jcmaster.c:1102-1105)
SWITCH_SETS_12 = [
    ["-precision", "12", "-sample", "1x1", "-quality", "75", "-notrellis", "-noovershoot", "-baseline"],      # config 5
    ["-precision", "12", "-quality", "75", "-notrellis", "-noovershoot", "-baseline"],                           # 4:2:0
    ["-precision", "12", "-quality", "90", "-notrellis", "-noovershoot", "-baseline", "-grayscale"],
    ["-precision", "12", "-quality", "60", "-notrellis", "-noovershoot", "-fastcrush", "-sample", "2x1"],
    ["-precision", "12", "-quality", "75", "-notrellis", "-noovershoot", "-fastcrush", "-restart", "1"],
    ["-precision", "12", "-quality", "100", "-notrellis", "-noovershoot", "-baseline", "-sample", "1x2"],
    # 12-bit on sampling layouts outside the tiled kernel's
    ["-precision", "12", "-quality", "75", "-notrellis", "-noovershoot", "-baseline", "-sample", "3x2"],
    ["-precision", "12", "-quality", "80", "-notrellis", "-noovershoot", "-fastcrush", "-sample", "4x1,1x1,2x1"],
    # 12-bit with the fast / float DCT (scaled divisors divided literally, jcdctmgr.c:332-336,646-678)
    ["-precision", "12", "-quality", "75", "-notrellis", "-noovershoot", "-baseline", "-dct", "fast"],
    ["-precision", "12", "-quality", "90", "-notrellis", "-noovershoot", "-baseline", "-dct", "float", "-sample", "2x1"],
    ["-precision", "12", "-quality", "60", "-notrellis", "-noovershoot", "-fastcrush", "-dct", "fast", "-sample", "3x2"],
]
SYNTH12 = [(21, 16, 16), (22, 33, 17), (23, 200, 136), (24, 640, 480), (25, 1, 1)]
SYNTH = [(11, 16, 16), (12, 33, 17), (13, 200, 136), (14, 640, 480), (15, 1, 1), (16, 8, 8), (17, 1920, 1080)]


def _key(image, sw):
    return json.dumps([image, sw])


# BASELINE.json's configurations at their stated sizes (a separate fixture: each case costs the reference seconds to a
# minute).  Images [seed, w, h] or [seed, w, h, 12]; seeds 1000.. are bench.py's first-rank inputs.
FULLSIZE = [
    ([300, 3840, 2160], ["-baseline", "-quality", "75", "-sample", "2x2"]),          # configs[1]
    ([1000, 3840, 2160], ["-baseline", "-quality", "75", "-sample", "2x2"]),
    ([300, 3840, 2160], ["-fastcrush", "-quality", "75", "-sample", "2x2"]),         # configs[2]
    ([1000, 3840, 2160], ["-fastcrush", "-quality", "75", "-sample", "2x2"]),
    ([17, 1920, 1080], ["-baseline", "-quality", "50", "-sample", "2x2"]),           # configs[3] sweep (q75 is in golden.json)
    ([17, 1920, 1080], ["-baseline", "-quality", "90", "-sample", "2x2"]),
    ([1001, 1920, 1080], ["-baseline", "-quality", "50", "-sample", "2x2"]),
    ([1001, 1920, 1080], ["-baseline", "-quality", "75", "-sample", "2x2"]),
    ([1001, 1920, 1080], ["-baseline", "-quality", "90", "-sample", "2x2"]),
    ([26, 3840, 2160, 12], ["-precision", "12", "-sample", "1x1", "-quality", "75", "-notrellis", "-noovershoot", "-baseline"]),   # configs[4]
    ([1000, 3840, 2160, 12], ["-precision", "12", "-sample", "1x1", "-quality", "75", "-notrellis", "-noovershoot", "-baseline"]),
    ([300, 3840, 2160], ["-quality", "75", "-sample", "2x2"]),                       # the library default (scan search) at 4K
]


def fullsize():
    from mozjpeg_b200.synth import synth_image12
    path = os.path.join(GOLD, "fullsize_golden.json")
    have = {}
    if "--force" not in sys.argv and os.path.exists(path):
        for c in json.load(open(path))["cases"]:
            have[_key(c["image"], c["switches"])] = c
    cases = []
    for image, sw in FULLSIZE:
        if _key(image, sw) in have:
            cases.append(have[_key(image, sw)]); continue
        im = synth_image12(*image[:3]) if len(image) > 3 else O.synth_image(*image)
        a = O.ref_encode(im, sw)
        cases.append({"image": image, "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
        print(image, sw, len(a), flush=True)
    json.dump({"generator": "tools/make_golden.py --fullsize", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref", "cases": cases},
              open(path, "w"), indent=0)
    print("wrote", len(cases), "full-size cases")


def colorspaces():
    """tests/golden/colorspace_golden.json: CMYK / YCCK / YCbCr->gray / JCS_UNKNOWN encodes by the reference (through
    build/librefcs.so, tests/refcs.c), raw-data input with 4 planes, and jpegtran on CMYK / YCCK sources."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import colorspace_cases as CC
    path = CC.GOLDEN
    if os.path.exists(path) and "--force" not in sys.argv:
        sys.exit(f"{path} exists; pass --force to overwrite it")
    if not CC.have_reference():
        sys.exit("build/librefcs.so is missing: run __graft_entry__.build() with the reference build under oracle/_ref/")
    cases = []
    for c in CC.pixel_cases():
        a = CC.reference_file(c)
        cases.append(dict(c, md5=CC.md5(a), size=len(a)))
    raw = []
    for conv, (in_cs, jcs) in CC.RAW_CONVERSIONS.items():
        for sw in CC.RAW_SETS:
            p = cjpeg.params_from_switches(sw, 227, 149, 4, in_cs, jcs)
            planes = CC.raw_planes(5, p, 4)
            a = CC.ref_encode(None, in_cs, 4, jcs, sw, planes=planes, size=(227, 149))
            raw.append(dict(id=CC.case_id(conv, " ".join(sw)), conv=conv, switches=sw, seed=5, w=227, h=149, md5=CC.md5(a), size=len(a)))
    tran = []
    for src in CC.TRAN_SOURCES:
        data = CC.tran_source(src)
        for sw in CC.TRAN_SETS + [["-grayscale"]]:
            r = subprocess.run([os.path.join(CC.REF, "jpegtran"), *sw], input=data, capture_output=True)
            rec = dict(id=CC.case_id(src, " ".join(sw)), source=src, switches=sw, source_md5=CC.md5(data))
            if r.returncode != 0 or not r.stdout:
                rec["error"] = r.stderr.decode().strip()
            else:
                rec.update(md5=CC.md5(r.stdout), size=len(r.stdout))
            tran.append(rec)
    json.dump({"generator": "tools/make_golden.py --colorspaces", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "cases": cases, "raw": raw, "transcode": tran}, open(path, "w"), indent=0)
    print("wrote", len(cases), "pixel,", len(raw), "raw-data and", len(tran), "jpegtran cases")

# per-image quantization tables (Encoder.encode_batch(..., qtables=)): every case is a batch of same-shaped images that
# share the base switches; image i adds its own table switches.  With -sample given explicitly the per-image parameter
# blocks differ in their tables only (cjpeg's -quality >= 80 would otherwise change the sampling factors).
PERIMAGE_Q = [
    # (seed, w, h, base switches, per-image table switches, extension parameters)
    (61, 227, 149, ["-baseline", "-sample", "2x2"], [["-quality", q] for q in ("30", "50", "75", "90", "95", "60")], None),
    (62, 1000, 664, ["-fastcrush", "-sample", "2x2"], [["-quality", q] for q in ("40", "85", "75", "20", "95")], None),
    (63, 227, 149, ["-sample", "2x2"], [["-quality", q] for q in ("50", "90", "75", "35")], None),
    (64, 227, 149, ["-baseline", "-sample", "2x1"], [["-quality", q] for q in ("60", "80", "45", "92")],
     {"trellis_q_opt": 1, "trellis_eob_opt": 1, "use_scans_in_trellis": 1}),
    (65, 227, 149, ["-dct", "fast", "-baseline", "-sample", "2x2"], [["-quality", q] for q in ("40", "75", "95", "55")], None),
    (66, 227, 149, ["-dct", "float", "-fastcrush", "-sample", "1x1"], [["-quality", q] for q in ("50", "90", "70", "25", "80")], None),
    (67, 227, 149, ["-baseline", "-sample", "2x2", "-smooth", "30"], [["-quality", q] for q in ("50", "85", "70", "30")], None),
    (68, 227, 149, ["-baseline", "-sample", "2x2", "-restart", "1"], [["-quality", q] for q in ("45", "75", "90", "65", "20", "99")], None),
    (69, 227, 149, ["-baseline", "-grayscale", "-sample", "1x1"], [["-quality", q] for q in ("30", "60", "90", "75")], None),
    (70, 1000, 664, ["-baseline", "-sample", "2x2"], [["-quality", "75"], ["-qtables", "@GOLD/qtables_a.txt"], ["-quality", "50"], ["-qtables", "@GOLD/qtables_a.txt", "-quality", "40"]], None),
    ([71, 12], 227, 149, ["-precision", "12", "-notrellis", "-noovershoot", "-fastcrush", "-sample", "2x2"], [["-quality", q] for q in ("1", "3", "50", "10", "90")], None),
    (72, 227, 149, ["-revert", "-sample", "2x2"], [["-quality", "1"], ["-quality", "1", "-baseline"], ["-quality", "5"], ["-quality", "30", "-baseline"], ["-quality", "2"]], None),
    # refused on the device: with the trellis on, a table holding 1 and 32767 is beyond the device divider
    (73, 227, 149, ["-fastcrush", "-sample", "2x2"], [["-quality", "75"], ["-quality", "50"], ["-qtables", "@GOLD/qtables_wide.txt"], ["-quality", "90"]], None),
]


def perimage_image(seed, w, h, i):
    """Image i of a per-image-table case: seeds count up from the case's; [seed, 12] = 12-bit samples."""
    if isinstance(seed, list):
        from mozjpeg_b200.synth import synth_image12
        return synth_image12(seed[0] + i, w, h)
    return O.synth_image(seed + i, w, h)


def perimage_q():
    """tests/golden/perimage_q_golden.json: per case and image the reference's file for base + that image's switches."""
    path = os.path.join(GOLD, "perimage_q_golden.json")
    if os.path.exists(path) and "--force" not in sys.argv:
        sys.exit(f"{path} exists; pass --force to overwrite it")
    expand = lambda sw: [os.path.join(GOLD, x[6:]) if x.startswith("@GOLD/") else x for x in sw]
    cases = []
    for seed, w, h, base, per_image, ext in PERIMAGE_Q:
        files = []
        for i, isw in enumerate(per_image):
            a = O.ref_encode(perimage_image(seed, w, h, i), expand(base + isw), ext)
            files.append({"switches": isw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
        cases.append({"seed": seed, "width": w, "height": h, "switches": base, "ext": ext, "images": files})
        print(seed, w, h, base, [f["size"] for f in files], flush=True)
    json.dump({"generator": "tools/make_golden.py --perimage-q", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "cases": cases}, open(path, "w"), indent=0)
    print("wrote", len(cases), "per-image-table cases")


def lossless():
    """tests/golden/lossless_golden.json: every case of tests/test_lossless.py (lossless mode at 8, 12 and 16 bits) encoded
    by the reference library through build/librefll.so (tests/refll.c).  Wherever the reference's own cjpeg binary can
    express the case (grayscale or RGB input read from a PGM / PPM whose maxval is the precision's largest sample, no
    hand-made script), the binary's bytes must equal the driver's."""
    import tempfile
    import zlib
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_lossless as T
    from mozjpeg_b200 import _abi as A
    cases, checked = [], 0
    for c in T.CASES:
        sw, cs, nc, prec, (h, w), kind, script = c
        pix = T.image(zlib.crc32(T._id(c).encode()), h, w, nc, prec, kind)
        a = T.ref_encode(pix, sw, cs, script)
        if cs in (A.CS_GRAYSCALE, A.CS_RGB) and script is None and int(pix.max()) <= (1 << prec) - 1:
            with tempfile.NamedTemporaryFile(suffix=".pnm") as f:
                f.write(b"%s\n%d %d\n%d\n" % (b"P5" if nc == 1 else b"P6", w, h, (1 << prec) - 1))
                f.write(pix.astype(">u2").tobytes() if prec > 8 else pix.tobytes())
                f.flush()
                b = O.ref_cjpeg(f.name, sw)
            assert a == b, ("refll disagrees with cjpeg", sw)
            checked += 1
        cases.append({"id": T._id(c), "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    json.dump({"generator": "tools/make_golden.py --lossless", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "cjpeg_binary_checked": checked, "cases": cases}, open(os.path.join(GOLD, "lossless_golden.json"), "w"), indent=0)
    print("wrote", len(cases), "lossless cases;", checked, "checked against the cjpeg binary")


def yuv():
    """tests/golden/yuv_golden.json: the reference's tj3EncodeYUVPlanes8 (oracle/_ref/libturbojpeg_ref.so through ctypes)
    on every subsampling x pixel format x size x plane stride of tests/yuv_cases.py: the md5 of every plane's pw x ph
    samples, or the reference's refusal."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import yuv_cases as Y
    ref = Y.RefTJ()
    cases = []
    for size in Y.SIZES:
        for pf in Y.PIXEL_FORMATS:
            pix = Y.case_pixels(size, pf)
            for ss in Y.SUBSAMPS:
                for pad in Y.PADS:
                    planes, err = ref.encode_planes(pix, pf, ss, pad)
                    c = {"size": Y.size_id(size), "pf": pf, "subsamp": ss, "pad": pad}
                    if err is not None:
                        c["error"] = err
                    else:
                        c["dims"] = [list(p.shape[::-1]) for p in planes]
                        c["md5"] = [Y.md5(p) for p in planes]
                    cases.append(c)
    ref.close()
    json.dump({"generator": "tools/make_golden.py --yuv", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "cases": cases}, open(os.path.join(GOLD, "yuv_golden.json"), "w"), indent=0)
    print("wrote", len(cases), "YUV cases;", sum("error" in c for c in cases), "refusals")


def decode():
    """tests/golden/decode_golden.json: for every source of tests/decode_cases.py, the md5 of the file and of the
    reference's jpeg_read_coefficients planes for it (oracle/_ref/librefshim.so through ctypes)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import decode_cases as D
    cases = []
    for c in D.CASES:
        src, _ = D.source(c)
        ref = O.ref_read_coefs(src)["coefs"]
        cases.append({"id": c[0], "src_md5": hashlib.md5(src).hexdigest(), "coef_md5": D.md5_planes(ref)})
    for name in D.EXTRA_IDS:
        src = D.extra_source(name)
        ref = O.ref_read_coefs(src)["coefs"]
        cases.append({"id": name, "src_md5": hashlib.md5(src).hexdigest(), "coef_md5": D.md5_planes(ref)})
    json.dump({"generator": "tools/make_golden.py --decode", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "cases": cases}, open(os.path.join(GOLD, "decode_golden.json"), "w"), indent=0)
    print("wrote", len(cases), "decode cases")


def transform():
    """tests/golden/transform_golden.json: the reference's own jpegtran on the sources of tests/transform_cases.py, per
    case the output's md5, size, SOF fields and component tables, or the reference's refusal."""
    import subprocess
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import transform_cases as X
    srcs = {sid: X.source(sid)[0] for sid in X.source_ids()}

    def run(cid, sid, sw):
        rec = {"id": cid, "source": sid, "switches": sw}
        r = subprocess.run([os.path.join(O.REF_DIR, "jpegtran"), *sw], input=srcs[sid], capture_output=True)
        if r.returncode != 0:
            msg = r.stderr.decode().strip().splitlines()[0] if r.stderr else f"exit {r.returncode}"
            rec["error"] = msg.replace(os.path.join(O.REF_DIR, "jpegtran"), "jpegtran")
            return rec
        w, h, comps, qmd5 = X.sof_dqt(r.stdout)
        rec.update(md5=X.md5(r.stdout), size=len(r.stdout), sof=[w, h, comps], qt_md5=qmd5)
        return rec

    cases = [run(*c) for c in X.main_matrix() + X.other_cases()]
    cases += [run(f"mixed_{sid}", sid, ["-rotate", "90"]) for sid in X.mixed_ids()]
    cases += [run(f"prog_{'_'.join(a.lstrip('-') for a in sw)}", "prog_420", sw) for sw in (["-rotate", "90"], ["-crop", "64x48+5+3", "-transpose"])]
    refusals = [run(f"refuse{k}", sid, sw) for k, (sid, sw) in enumerate(X.REFUSALS)]
    json.dump({"generator": "tools/make_golden.py --transform", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "sources": {sid: X.md5(b) for sid, b in srcs.items()}, "cases": cases, "refusals": refusals},
              open(os.path.join(GOLD, "transform_golden.json"), "w"), indent=0)
    print("wrote", len(cases), "transform cases,", sum("error" in c for c in cases), "refused;", len(refusals), "refusals")


def recompress():
    """tests/golden/recompress_golden.json: for every source of tests/recompress_cases.py the md5 of the file and of the
    pixels the reference decodes from it (build/librefdec.so: jpeg_read_scanlines of a default decompress object), and
    for every (source, switches) of its RECOMPRESS list the md5 and size of what the reference's cjpeg writes."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import recompress_cases as R
    if not R.have_reference():
        sys.exit("build/librefdec.so or oracle/_ref/cjpeg is missing: run __graft_entry__.build() with the reference build under oracle/_ref/")
    cases = []
    for sid in R.all_ids():
        src, _ = R.source(sid)
        px, info = R.ref_decompress(src)
        cases.append({"id": sid, "src_md5": R.md5(src), "pix_md5": R.md5(px), "shape": list(px.shape), "out_color_space": info[3], "warnings": info[5]})
    rec = []
    for sid, sw in R.RECOMPRESS:
        out = R.ref_cjpeg(R.source(sid)[0], sw)
        rec.append({"source": sid, "switches": sw, "md5": R.md5(out), "size": len(out)})
    json.dump({"generator": "tools/make_golden.py --recompress", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "cases": cases, "recompress": rec}, open(os.path.join(GOLD, "recompress_golden.json"), "w"), indent=0)
    print("wrote", len(cases), "decompress cases,", len(rec), "recompress cases")


def decompress_options():
    """tests/golden/decompress_options_golden.json: for every (source, options) of tests/decompress_options_cases.py the
    md5 of the source, the fields jpeg_calc_output_dimensions sets and the md5 of the pixels the reference decodes with
    those options (build/librefdecopt.so), and the reference's message for each refused colour pair."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import decompress_options_cases as O
    if not O.have_reference():
        sys.exit("build/librefdecopt.so is missing: run __graft_entry__.build() with the reference build under oracle/_ref/")
    cases = []
    for cid, sid, scale, dct, fancy, cs in O.cases():
        src, _ = O.source(sid)
        px, info, msg = O.ref_decompress(src, O.opts_tuple(scale, dct, fancy, cs))
        if px is None:
            sys.exit(f"{cid}: the reference refuses it: {msg}")
        nc = info[6]
        cases.append({"id": cid, "src_md5": O.md5(src), "pix_md5": O.md5(px), "shape": list(px.shape), "out_color_space": info[3],
                      "components": [info[7 + 3 * c:10 + 3 * c] for c in range(nc)], "warnings": info[5]})
    refused = []
    for sid, cs in O.REFUSED_PAIRS:
        _, _, msg = O.ref_decompress(O.source(sid)[0], (1, 1, 0, 1, cs), header_only=True)
        refused.append({"source": sid, "out_color_space": cs, "message": msg})
    json.dump({"generator": "tools/make_golden.py --decompress-options", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref",
               "cases": cases, "refused_pairs": refused}, open(os.path.join(GOLD, "decompress_options_golden.json"), "w"), indent=0)
    print("wrote", len(cases), "cases,", len(refused), "refused pairs")


def main():
    if "--decompress-options" in sys.argv:
        return decompress_options()
    if "--recompress" in sys.argv:
        return recompress()
    if "--transform" in sys.argv:
        return transform()
    if "--decode" in sys.argv:
        return decode()
    if "--yuv" in sys.argv:
        return yuv()
    if "--lossless" in sys.argv:
        return lossless()
    if "--perimage-q" in sys.argv:
        return perimage_q()
    if "--fullsize" in sys.argv:
        return fullsize()
    if "--colorspaces" in sys.argv:
        return colorspaces()
    os.makedirs(GOLD, exist_ok=True)
    # cases already recorded are kept as they are unless --force is given (a full regeneration takes a while)
    have = {}
    if "--force" not in sys.argv and os.path.exists(os.path.join(GOLD, "golden.json")):
        for c in json.load(open(os.path.join(GOLD, "golden.json")))["cases"]:
            have[_key(c["image"], c["switches"])] = c
    shutil.copyfile(os.path.join(REF, "testimages", "testorig.ppm"), os.path.join(GOLD, "testorig.ppm"))
    cases = []
    ppm = os.path.join(GOLD, "testorig.ppm")
    w, h, nc, data = cjpeg.read_ppm(open(ppm, "rb").read())
    img = np.frombuffer(data, dtype=np.uint8).reshape(h, w, nc)
    for sw in SWITCH_SETS:
        if _key("testorig", sw) in have: cases.append(have[_key("testorig", sw)]); continue
        a = O.ref_cjpeg(ppm, sw)                   # the reference's own cjpeg binary
        b = O.ref_encode(img, sw)                  # our driver around the reference library
        assert a == b, ("refshim disagrees with cjpeg", sw)
        cases.append({"image": "testorig", "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    for sw in CJPEG_ONLY:
        a = O.ref_cjpeg(ppm, sw)
        cases.append({"image": "testorig", "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    for sw in SWITCH_SETS_EXTRA:
        a = O.ref_cjpeg(ppm, sw)
        cases.append({"image": "testorig", "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    expand = lambda sw: [os.path.join(GOLD, x[6:]) if x.startswith("@GOLD/") else x for x in sw]
    for sw in SWITCH_SETS_FILES:
        a = O.ref_cjpeg(ppm, expand(sw))
        cases.append({"image": "testorig", "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    for (seed, sw_, sh_) in SYNTH[:4]:
        im = O.synth_image(seed, sw_, sh_)
        for sw in SWITCH_SETS_FILES:
            a = O.ref_encode(im, expand(sw))
            cases.append({"image": [seed, sw_, sh_], "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    # maximum dimensions (JPEG_MAX_DIMENSION 65500, jmorecfg.h): one block row / one block column
    for (seed, sw_, sh_) in [(18, 65500, 3), (19, 3, 65500)]:
        im = O.synth_image(seed, sw_, sh_)
        for sw in (["-baseline", "-quality", "75"], ["-quality", "75"], ["-fastcrush", "-quality", "75", "-sample", "2x2"], ["-revert", "-restart", "1"],
                   ["-baseline", "-quality", "85", "-sample", "1x1"], ["-baseline", "-grayscale", "-quality", "75"], ["-revert", "-sample", "2x1", "-optimize"],
                   ["-baseline", "-quality", "75", "-restart", "1"], ["-dct", "float", "-baseline", "-quality", "75"], ["-baseline", "-quality", "75", "-smooth", "30"]):
            if _key([seed, sw_, sh_], sw) in have: cases.append(have[_key([seed, sw_, sh_], sw)]); continue
            a = O.ref_encode(im, sw)
            cases.append({"image": [seed, sw_, sh_], "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    for (seed, sw_, sh_) in SYNTH:
        im = O.synth_image(seed, sw_, sh_)
        sets = SWITCH_SETS + SWITCH_SETS_EXTRA if sw_ * sh_ <= 640 * 480 else [s for s in SWITCH_SETS if s in (["-revert", "-dct", "int"], ["-baseline", "-quality", "75", "-sample", "2x2"], ["-fastcrush", "-quality", "75", "-sample", "2x2"], ["-baseline", "-quality", "90", "-sample", "2x2"], ["-quality", "75"])]
        for sw in sets:
            if _key([seed, sw_, sh_], sw) in have: cases.append(have[_key([seed, sw_, sh_], sw)]); continue
            a = O.ref_encode(im, sw)
            cases.append({"image": [seed, sw_, sh_], "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    from mozjpeg_b200.synth import synth_image12
    for (seed, sw_, sh_) in SYNTH12:
        im = synth_image12(seed, sw_, sh_)
        for sw in SWITCH_SETS_12:
            if _key([seed, sw_, sh_, 12], sw) in have: cases.append(have[_key([seed, sw_, sh_, 12], sw)]); continue
            a = O.ref_encode(im, sw)
            cases.append({"image": [seed, sw_, sh_, 12], "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    # raw-data input (jpeg_write_raw_data): separate fixture, the inputs are component planes
    from mozjpeg_b200.synth import synth_planes
    raw_cases = []
    for (seed, w_, h_) in [(31, 33, 17), (32, 200, 136), (33, 227, 149), (34, 640, 480)]:
        for sw in (["-baseline", "-quality", "75"], ["-quality", "75"], ["-baseline", "-quality", "85", "-sample", "1x1"],
                   ["-fastcrush", "-quality", "60", "-sample", "2x1"], ["-baseline", "-quality", "75", "-grayscale"],
                   ["-baseline", "-notrellis", "-quality", "90", "-sample", "1x2", "-dct", "float"],
                   ["-baseline", "-quality", "75", "-sample", "4x2"], ["-fastcrush", "-quality", "70", "-sample", "2x2,1x1,2x2"]):
            pp = cjpeg.params_from_switches(sw, w_, h_, 1 if "-grayscale" in sw else 3)
            a = O.ref_encode_raw(synth_planes(pp, seed), w_, h_, sw)
            raw_cases.append({"seed": seed, "width": w_, "height": h_, "switches": sw, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    json.dump({"generator": "tools/make_golden.py", "cases": raw_cases}, open(os.path.join(GOLD, "raw_golden.json"), "w"), indent=0)
    # coefficient-domain re-encode (jpegtran = jpeg_read_coefficients + jpeg_write_coefficients): the source file is
    # what the reference's encoder makes of (seed, size, enc switches); the md5 is what the reference's own jpegtran
    # binary writes for (tran switches), its keep-the-smaller-file rule (jpegtran.c:772-775) included
    tr_cases = []
    for (seed, w_, h_) in [(41, 33, 17), (42, 200, 136), (43, 1, 1), (44, 640, 480)]:
        im = O.synth_image(seed, w_, h_)
        for esw in (["-revert"], ["-quality", "75"], ["-baseline", "-quality", "85", "-sample", "1x1"], ["-revert", "-grayscale", "-progressive"],
                    ["-fastcrush", "-quality", "60", "-sample", "2x1"], ["-revert", "-sample", "3x2"]):
            srcfile = O.ref_encode(im, esw)
            for tsw in ([], ["-revert"], ["-optimize"], ["-progressive"], ["-fastcrush"], ["-revert", "-optimize"], ["-revert", "-progressive"],
                        ["-restart", "1"], ["-fastcrush", "-restart", "2B"], ["-progressive", "-fastcrush"], ["-copy", "none", "-progressive", "-restart", "1"]):
                a = O.ref_jpegtran(srcfile, tsw)
                tr_cases.append({"seed": seed, "width": w_, "height": h_, "enc": esw, "tran": tsw, "md5": hashlib.md5(a).hexdigest(), "size": len(a),
                                 "src_md5": hashlib.md5(srcfile).hexdigest()})
    json.dump({"generator": "tools/make_golden.py", "cases": tr_cases}, open(os.path.join(GOLD, "transcode_golden.json"), "w"), indent=0)
    # extension parameters cjpeg has no switch for (jpeg_c_set_*_param): use_scans_in_trellis / trellis_freq_split
    ext_cases = []
    for (seed, w_, h_) in [(51, 33, 17), (52, 200, 136), (53, 640, 480), (54, 1, 1)]:
        im = O.synth_image(seed, w_, h_)
        for sw in (["-baseline", "-quality", "75"], ["-fastcrush", "-quality", "75"], ["-quality", "75"], ["-baseline", "-quality", "90", "-sample", "1x1"],
                   ["-fastcrush", "-quality", "50", "-grayscale"], ["-baseline", "-quality", "80", "-restart", "1", "-sample", "2x1"],
                   ["-fastcrush", "-quality", "30", "-sample", "1x1"]):
            for ext in ({"use_scans_in_trellis": 1}, {"use_scans_in_trellis": 1, "trellis_freq_split": 3}, {"use_scans_in_trellis": 1, "trellis_freq_split": 20},
                        {"trellis_num_loops": 2}, {"trellis_num_loops": 3, "use_scans_in_trellis": 1},
                        {"trellis_q_opt": 1}, {"trellis_q_opt": 1, "trellis_num_loops": 2}, {"trellis_q_opt": 1, "trellis_num_loops": 3, "use_scans_in_trellis": 1},
                        {"trellis_eob_opt": 1}, {"trellis_eob_opt": 1, "use_scans_in_trellis": 1}, {"trellis_eob_opt": 1, "trellis_q_opt": 1, "trellis_num_loops": 2}):
                a = O.ref_encode(im, sw, ext)
                ext_cases.append({"seed": seed, "width": w_, "height": h_, "switches": sw, "ext": ext, "md5": hashlib.md5(a).hexdigest(), "size": len(a)})
    json.dump({"generator": "tools/make_golden.py", "cases": ext_cases}, open(os.path.join(GOLD, "ext_golden.json"), "w"), indent=0)
    assert cases[0]["md5"] == "9a68f56bc76e466aa7e52f415d0f4a5f", "reference build does not reproduce MD5_JPEG_420_ISLOW"
    json.dump({"generator": "tools/make_golden.py", "reference": "mozilla/mozjpeg 5.0.0 (C path, WITH_SIMD=0), oracle/_ref", "cases": cases},
              open(os.path.join(GOLD, "golden.json"), "w"), indent=0)
    print("wrote", len(cases), "cases")


if __name__ == "__main__":
    main()
