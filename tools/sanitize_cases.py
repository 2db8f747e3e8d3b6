#!/usr/bin/env python3
"""Small encodes that together launch every kernel family (run under compute-sanitizer by tools/sanitize.sh)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import mozjpeg_b200 as mj
from mozjpeg_b200.synth import synth_image, synth_image12, synth_planes

enc = mj.Encoder(0)
w, h = 203, 141
img = np.stack([synth_image(s, w, h) for s in range(2)])
cases = [["-baseline", "-quality", "75", "-sample", "2x2"],          # forward (TMA + bulk stores), trellis classes, DC trellis, sequential coder
         ["-baseline", "-quality", "95", "-sample", "1x1"],          # dense blocks: the 32-entry and generic trellis classes
         ["-fastcrush", "-quality", "75"],                           # progressive coder, EOBRUN kernels
         ["-quality", "75"],                                         # scan search (64 candidates), Al selection
         ["-baseline", "-quality", "75", "-restart", "1"],           # restart intervals
         ["-baseline", "-quality", "75", "-smooth", "20"],           # smoothing pre-pass
         ["-baseline", "-quality", "75", "-sample", "3x2"],          # generic forward kernel
         ["-dct", "float", "-baseline", "-quality", "75"], ["-dct", "fast", "-baseline", "-quality", "75"],
         ["-revert"], ["-baseline", "-grayscale", "-quality", "75"],
         ["-scans", os.path.join(ROOT, "tests", "golden", "scans_b.txt"), "-quality", "80"]]   # two sequential scans: per-scan statistics from the symbol records
n = 0
for sw in cases:
    p = mj.params_from_switches(sw, w, h)
    out = enc.encode_batch(p, img); n += len(out)
    assert all(o[:2] == b"\xff\xd8" and o[-2:] == b"\xff\xd9" for o in out), sw
# optional trellis modes: band kernel, EOB-run rows, table re-fitting
for ext in ({"use_scans_in_trellis": 1}, {"trellis_eob_opt": 1}, {"trellis_q_opt": 1, "trellis_num_loops": 2}):
    p = mj.params_from_switches(["-baseline", "-quality", "75"], w, h)
    for k, v in ext.items():
        setattr(p, k, v)
    n += len(enc.encode_batch(p, img))
# 12-bit, raw-data input, coefficient input (import kernel), a pixel order with 4 samples
p = mj.params_from_switches(["-precision", "12", "-quality", "75", "-notrellis", "-noovershoot", "-baseline"], w, h)
n += len(enc.encode_batch(p, np.stack([synth_image12(3, w, h)])))
p = mj.params_from_switches(["-baseline", "-quality", "75"], w, h)
n += len(enc.encode_batch_raw(p, [a[None] for a in synth_planes(p, 5)]))
q = mj.params_from_switches(["-baseline", "-quality", "75"], w, h)
q.in_color_space, q.input_components = 13, 4                        # JCS_EXT_BGRA
n += len(enc.encode_batch(q, np.concatenate([img[..., ::-1], img[..., :1]], axis=-1)))
# per-image quantization tables: one 1024-pixel-wide image at three qualities (image stride 0: one TMA tensor map that
# every image addresses as image 0), a mixed batch at that width (TMA with per-image sets) and one at 203 (per-thread
# loads), and raw-data / coefficient input shared by every image (zero plane stride, staged once)
wide = np.stack([synth_image(s, 1024, 64) for s in range(2)])
pw = mj.params_from_switches(["-baseline", "-quality", "75", "-sample", "2x2"], 1024, 64)
n += len(enc.encode_batch(pw, wide[:1], qtables=mj.quality_tables(pw, (30, 60, 90))))
n += len(enc.encode_batch(pw, wide, qtables=mj.quality_tables(pw, (20, 95))))
p = mj.params_from_switches(["-baseline", "-quality", "75", "-sample", "2x2"], w, h)
n += len(enc.encode_batch(mj.params_from_switches(["-quality", "75"], w, h), img, qtables=mj.quality_tables(p, (20, 95))))
n += len(enc.encode_batch_raw(p, [a[None] for a in synth_planes(p, 6)], qtables=mj.quality_tables(p, (30, 60, 90))))
pc = mj.params_from_switches(["-revert", "-quality", "75"], w, h)
n += len(enc.encode_batch_coefs(pc, [np.zeros((1, (h + 15) // 16 * (2 if ci == 0 else 1), (w + 15) // 16 * (2 if ci == 0 else 1), 64), np.int16) for ci in range(3)],
                                qtables=mj.quality_tables(pc, (30, 60, 90))))
# an interior-tile-rich frame for the TMA path and a wide one
big = np.stack([synth_image(9, 1024, 256)])
n += len(enc.encode_batch(mj.params_from_switches(["-baseline", "-quality", "75", "-sample", "2x2"], 1024, 256), big))
print("sanitize cases done:", n, "files, kernel launches", enc.kernel_launches())
enc.close()
