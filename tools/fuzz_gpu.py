#!/usr/bin/env python3
"""Randomised device-vs-oracle cross-check (runs on a GPU box): random shapes, cjpeg switch sets, extension parameters
(the optional trellis modes), pixel orders of the RGB family, the CMYK / YCCK / YCbCr->gray / JCS_UNKNOWN conversions and small batches (some with
per-image quantization tables) through the C-ABI, every file compared
byte for byte with the CPU oracle (itself pinned to the reference).  Test infrastructure.
usage: fuzz_gpu.py [--yuv | --content] [seed] [cases] [seconds]      (exit status 1 if anything differs)"""
import os, random, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np
from oracle import oracle as O
import mozjpeg_b200 as mj
from mozjpeg_b200 import _abi as A
from mozjpeg_b200.synth import synth_image12
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import colorspace_cases as CC       # CMYK / YCCK / YCbCr->gray / JCS_UNKNOWN conversions and their restatement


def fuzz_yuv(seed, cases, budget):
    """fuzz_gpu.py --yuv [seed] [cases] [seconds]: tj3EncodeYUVPlanes8 on the device against the reference library
    (oracle/_ref/libturbojpeg_ref.so) for random shapes, subsamplings, pixel formats, source pitches, plane pitches and
    small batches, every plane byte for byte and every pitch / gap byte untouched."""
    import yuv_cases as Y
    rng = random.Random(seed)
    ref = Y.RefTJ()
    bad = tot = refused = 0
    t0 = time.time()
    for it in range(cases):
        if time.time() - t0 > budget:
            break
        w = rng.choice([1, 2, 3, 5, 7, 8, 15, 16, 17, 31, 33, 63, 100, 255, 256, 257, 300, 513, 1023])
        h = rng.choice([1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 33, 64, 99, 200])
        ss, pf = rng.choice(Y.SUBSAMPS), rng.choice([f for f in Y.PIXEL_FORMATS if f != "CMYK"])
        if pf == "GRAY" and ss != "gray":
            refused += 1; continue
        n = rng.choice([1, 1, 2, 3, 5])
        ps = Y.PIXEL_FORMATS[pf]
        imgs = [Y.to_pixel_format(Y.synth_rgb(rng.randrange(1 << 20), w, h), pf, rng.randrange(1 << 20)) for _ in range(n)]
        row_pitch = w * ps + rng.choice([0, 0, 1, 3, 16])
        image_stride = row_pitch * h + rng.choice([0, 5, 64])
        src = np.zeros(image_stride * n + 16, np.uint8)
        off = rng.choice([0, 0, 1, 7])                    # unaligned first pixel
        for i, im in enumerate(imgs):
            for y in range(h):
                a = off + i * image_stride + y * row_pitch
                src[a: a + w * ps] = im[y].reshape(-1)
        cs = A.CS_GRAYSCALE if ss == "gray" else A.CS_YCbCr
        p = mj.tj3_params(w, h, subsamp=ss, pixel_format=pf, colorspace=cs)
        geo = [mj.yuv_plane_dims(p, ci) for ci in range(p.num_components)]
        pitch = [pw + rng.choice([0, 0, 1, 13, 64]) for pw, _ in geo]
        stride = [pt * ph + rng.choice([0, 3, 100]) for pt, (_, ph) in zip(pitch, geo)]
        pofs = [rng.choice([0, 0, 1, 5]) for _ in geo]
        outs = [np.full(st * n + 8, 0xEE, np.uint8) for st in stride]
        try:
            enc.encode_yuv_batch_ptr(p, src.ctypes.data + off, False, row_pitch, image_stride, [o.ctypes.data + po for o, po in zip(outs, pofs)],
                                     False, pitch, stride, n)
        except Exception as ex:
            bad += 1; print("YUV DEVICE FAIL", (w, h, n), ss, pf, ex); continue
        tot += 1
        for i, im in enumerate(imgs):
            want, err = ref.encode_planes(im, pf, ss)
            ok = err is None
            for ci, ((pw, ph), pt, st, po, o) in enumerate(zip(geo, pitch, stride, pofs, outs)):
                blk = o[po + i * st: po + i * st + pt * ph].reshape(ph, pt)
                ok = ok and np.array_equal(blk[:, :pw], want[ci]) and (blk[:, pw:] == 0xEE).all()
                ok = ok and (o[po + i * st + pt * ph: po + (i + 1) * st] == 0xEE).all() and (o[:po] == 0xEE).all()
            if not ok:
                bad += 1; print("YUV MISMATCH", (w, h, n), ss, pf, "image", i, (row_pitch, image_stride, off, pitch, stride, pofs)); break
    ref.close()
    print("yuv seed", seed, "bad", bad, "compared", tot, "refused", refused, "seconds %.0f" % (time.time() - t0))
    return bad


def fuzz_content(seed, cases, budget):
    """fuzz_gpu.py --content [seed] [cases] [seconds]: the constructed families of tests/adversarial_cases.py (flat-block
    ladders under random flat tables, basis-sum blocks, screen content) cropped at random, under random switch sets and
    sampling layouts, device against the CPU oracle."""
    import adversarial_cases as ADV
    rng = random.Random(seed)
    screens = list(ADV.screen_images(seed).values())
    bad = tot = refused = 0
    t0 = time.time()
    for it in range(cases):
        if time.time() - t0 > budget:
            break
        fam = rng.choice(["ladder", "basis", "screen"])
        qt = None
        if fam == "ladder":
            img = ADV.flat_ladder()
            qt = ADV.flat_tables([rng.randint(1, 255) for _ in range(rng.choice([1, 2, 5]))])
        elif fam == "basis":
            img = ADV.basis_image(rng.choice([6, 8, 12, 16, 24]), rng.randrange(1 << 20))
        else:
            img = rng.choice(screens)
        h, w = img.shape[:2]
        img = np.ascontiguousarray(img[:rng.randint(max(1, h - 9), h), :rng.randint(max(1, w - 9), w)])
        sw = rng.choice([["-baseline"], ["-baseline", "-notrellis"], ["-fastcrush"], [], ["-revert"], ["-baseline", "-restart", "1"]])
        sw = sw + ["-quality", str(rng.choice([30, 75, 95, 100]))] if rng.random() < 0.4 else list(sw)
        if rng.random() < 0.3: sw += ["-dct", rng.choice(["fast", "float"])]
        if img.ndim == 3: sw += rng.choice([["-sample", s] for s in ("1x1", "2x1", "1x2", "2x2", "3x2")] + [["-grayscale"]])
        try:
            p = mj.params_from_switches(sw, img.shape[1], img.shape[0], 1 if img.ndim == 2 else 3)
        except Exception:
            refused += 1; continue
        imgs = img[None]
        try:
            got = enc.encode_batch(p, imgs, qtables=qt)
        except mj.B200JpegError as ex:
            if ex.code == -2:
                refused += 1; continue
            bad += 1; print("CONTENT DEVICE FAIL", fam, sw, img.shape, ex); continue
        tot += 1
        for i, out in enumerate(got):
            pi = p
            if qt is not None:
                pi = p.copy(); np.ctypeslib.as_array(pi.quant_tbl)[:] = qt[i]
            if out != O.oracle_encode(pi, img).jpeg:
                bad += 1; print("CONTENT MISMATCH", fam, sw, img.shape, "table set", i); break
    print("content seed", seed, "bad", bad, "compared", tot, "refused", refused, "seconds %.0f" % (time.time() - t0))
    return bad


if "--content" in sys.argv:
    sys.argv.remove("--content")
    enc = mj.Encoder(0)
    nbad = fuzz_content(int(sys.argv[1]) if len(sys.argv) > 1 else 1, int(sys.argv[2]) if len(sys.argv) > 2 else 300,
                        float(sys.argv[3]) if len(sys.argv) > 3 else 120.0)
    enc.close()
    sys.exit(1 if nbad else 0)

if "--yuv" in sys.argv:
    sys.argv.remove("--yuv")
    enc = mj.Encoder(0)
    nbad = fuzz_yuv(int(sys.argv[1]) if len(sys.argv) > 1 else 1, int(sys.argv[2]) if len(sys.argv) > 2 else 2000,
                    float(sys.argv[3]) if len(sys.argv) > 3 else 300.0)
    enc.close()
    sys.exit(1 if nbad else 0)

seed = int(sys.argv[1]) if len(sys.argv) > 1 else 1
cases = int(sys.argv[2]) if len(sys.argv) > 2 else 300
budget = float(sys.argv[3]) if len(sys.argv) > 3 else 120.0
rng = random.Random(seed)
lib = A.load()
enc = mj.Encoder(0)
bad = tot = refused = 0
t0 = time.time()
for it in range(cases):
    if time.time() - t0 > budget:
        break
    w = rng.choice([1, 7, 8, 16, 17, 33, 64, 100, 131, 203, 256, 300, 513]); h = rng.choice([1, 5, 8, 16, 23, 40, 64, 77, 141, 200])
    sw = []
    twelve = rng.random() < 0.08
    prof = rng.choice(["", "-revert", "-baseline", "-baseline", "-fastcrush", "-progressive"])
    if prof == "-progressive": sw += ["-revert", "-progressive"] if rng.random() < 0.5 else ["-progressive"]
    elif prof: sw.append(prof)
    if rng.random() < 0.8: sw += ["-quality", str(rng.choice([5, 20, 40, 60, 75, 80, 85, 90, 95, 100]))]
    if rng.random() < 0.5: sw += ["-sample", rng.choice(["1x1", "2x1", "1x2", "2x2", "3x1", "4x2", "2x2,1x1,2x2", "4x1,1x1,2x1", "3x2"])]
    if rng.random() < 0.15 and not twelve: sw += ["-grayscale"]
    if rng.random() < 0.25: sw += ["-restart", rng.choice(["1", "2", "3B", "7B", "1B"])]
    if rng.random() < 0.15: sw += ["-dct", rng.choice(["fast", "float"])]
    if rng.random() < 0.1: sw += ["-smooth", str(rng.choice([1, 10, 50, 100]))]
    if twelve: sw = ["-precision", "12", "-notrellis", "-noovershoot"] + sw
    elif rng.random() < 0.15: sw += [rng.choice(["-notrellis", "-notrellis-dc", "-noovershoot", "-optimize"])]
    conv = rng.choice(list(CC.CONVERSIONS)) if rng.random() < 0.25 else None
    if conv and "-grayscale" in sw:
        sw.remove("-grayscale")
    in_cs, ic, jcs = CC.CONVERSIONS[conv] if conv else (A.CS_RGB, 3, None)
    try:
        p = mj.params_from_switches(sw, w, h, ic, in_cs, jcs)
    except Exception:
        continue
    ext = {}
    if p.trellis_quant and rng.random() < 0.35:
        if rng.random() < 0.5: ext["trellis_eob_opt"] = 1
        if rng.random() < 0.5: ext["trellis_q_opt"] = 1
        if rng.random() < 0.4: ext["use_scans_in_trellis"] = 1; ext["trellis_freq_split"] = rng.choice([1, 3, 8, 20, 62])
        if rng.random() < 0.4: ext["trellis_num_loops"] = rng.choice([2, 3])
    for k, v in ext.items():
        setattr(p, k, v)
    if lib.b200jpeg_validate(C.byref(p)) != 0:
        refused += 1
        continue
    n = rng.choice([1, 1, 2, 3])
    if conv:
        imgs = [CC.cmyk_image(rng.randrange(1 << 20), w, h, ic, 12 if twelve else 8) for _ in range(n)]
    else:
        imgs = [synth_image12(rng.randrange(1 << 20), w, h) if twelve else O.synth_image(rng.randrange(1 << 20), w, h) for _ in range(n)]
    # small batches sometimes carry per-image quantization tables (each image's reference: p with its tables)
    qt = None
    if n > 1 and rng.random() < 0.4:
        qt = mj.quality_tables(p, [rng.choice([1, 10, 30, 50, 75, 90, 100]) for _ in range(n)], force_baseline=rng.random() < 0.5)

    def with_tables(pp, i):
        if qt is None:
            return pp
        c = pp.copy(); np.ctypeslib.as_array(c.quant_tbl)[:] = qt[i]
        return c
    refs = [CC.oracle_encode(with_tables(p, i), im).jpeg for i, im in enumerate(imgs)]
    arr = np.stack(imgs)
    q = p
    order = None
    if rng.random() < 0.3 and not conv:
        order = rng.choice(list(A.CS_EXT))
        val, size, ro, go, bo = A.CS_EXT[order]
        out = np.random.default_rng(it).integers(0, 4096 if twelve else 256, arr.shape[:3] + (size,), dtype=arr.dtype)
        out[..., ro] = arr[..., 0]; out[..., go] = arr[..., 1]; out[..., bo] = arr[..., 2]
        arr = np.ascontiguousarray(out)
        q = mj.params_from_switches(sw, w, h, 3)
        for k, v in ext.items():
            setattr(q, k, v)
        q.in_color_space, q.input_components = val, size
        if lib.b200jpeg_validate(C.byref(q)) != 0:
            refused += 1
            continue
    try:
        got = enc.encode_batch(q, arr, qtables=qt)
    except mj.B200JpegError as ex:
        if ex.code == -2:                       # B200JPEG_ERR_UNSUPPORTED decided at encode time (e.g. fast / float DCT with a non-tiled sampling layout)
            refused += 1; continue
        bad += 1; print("DEVICE FAIL", sw, ext, order, (w, h, n), ex); continue
    except Exception as ex:
        bad += 1; print("DEVICE FAIL", sw, ext, order, (w, h, n), ex); continue
    tot += 1
    for i in range(n):
        if got[i] != refs[i]:
            bad += 1; print("MISMATCH", sw, ext, conv or order, (w, h, n), "image", i, len(got[i]), len(refs[i])); break
print("seed", seed, "bad", bad, "compared", tot, "refused", refused, "seconds %.0f" % (time.time() - t0))
enc.close()
sys.exit(1 if bad else 0)
