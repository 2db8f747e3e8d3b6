#!/usr/bin/env python3
"""Randomised device-vs-oracle cross-check (runs on a GPU box): random shapes, cjpeg switch sets, extension parameters
(the optional trellis modes), pixel orders of the RGB family, the CMYK / YCCK / YCbCr->gray / JCS_UNKNOWN conversions and small batches (some with
per-image quantization tables) through the C-ABI, every file compared
byte for byte with the CPU oracle (itself pinned to the reference).  Test infrastructure.
usage: fuzz_gpu.py [seed] [cases] [seconds]      (exit status 1 if anything differs)"""
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
