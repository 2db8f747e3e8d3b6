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
# device entropy decode: good sources, then the malformed ones it must refuse without reading or writing out of bounds
# (truncated segment, invalid code, wrong RSTn) and garbage after the last MCU, which it accepts
from mozjpeg_b200 import jpegtran as T
srcs = enc.encode_batch(mj.params_from_switches(["-revert", "-quality", "90"], w, h), img)
rst = enc.encode_batch(mj.params_from_switches(["-revert", "-quality", "90", "-restart", "1"], w, h), img[:1])[0]
n += len(T.transcode(enc, srcs, None, ["-optimize"]))
# lossless transforms in the coefficient import: partial edge iMCUs (rotations, transverse), crops, gray output, and
# caller planes in the source's geometry
for tsw in (["-rotate", "90"], ["-transverse"], ["-rotate", "180", "-crop", "64x48+5+3"], ["-grayscale", "-flip", "horizontal"]):
    n += len(T.transcode(enc, srcs, None, tsw))
n += len(T.transcode(enc, srcs[:1], enc.read_coefficients(srcs[:1]), ["-rotate", "270", "-trim"]))
n += len(enc.read_coefficients(srcs))
n += len(enc.read_coefficients([rst]))
sc = T.parse_source(srcs[0]).scans[0]
mid = sc.data_offset + sc.data_size // 2
k = rst.index(b"\xff\xd1", T.parse_source(rst).scans[0].data_offset)
for bad in (srcs[0][:mid], srcs[0][:mid] + b"\xff\x00" * 8 + srcs[0][mid + 16:], rst[:k + 1] + b"\xd5" + rst[k + 2:]):
    try:
        enc.read_coefficients([bad])
    except mj.B200JpegError as e:
        assert e.code == mj._abi.ERR_BAD_SOURCE, e
n += len(enc.read_coefficients([srcs[0][:sc.data_offset + sc.data_size] + bytes(range(1, 200)) + srcs[0][sc.data_offset + sc.data_size:]]))
# recompression (IDCT, upsampling + colour conversion, then the pixel encode): 4:2:0 at a ragged size
rag = enc.encode_batch(mj.params_from_switches(["-revert", "-quality", "90"], 203, 131), np.stack([synth_image(11, 203, 131), synth_image(12, 203, 131)]))
n += len(enc.recompress(mj.params_for_jpeg_input(["-baseline", "-quality", "75", "-sample", "2x2"], rag[0]), rag))
# decompression with options: the reduced IDCTs (1x1, 2x2, 4x4), ifast and float, plain upsampling, EXT_* layouts
for kw in (dict(scale=(1, 8)), dict(scale=(1, 4), dct="fast", fancy=False), dict(scale=(1, 2), dct="float", colorspace="bgrx"),
           dict(dct="fast", colorspace="gray"), dict(fancy=False, colorspace="xrgb")):
    n += len(enc.decompress(rag, **kw))
    n += len(enc.recompress(mj.params_for_jpeg_input(["-baseline", "-quality", "75"], rag[0], **kw), rag, **kw))
# every scale (all_scales): the scaled IDCTs of jidctint.c, one small ragged size per N, in the one-geometry form, the
# ragged form (a mixed batch of two geometries) and the PLANE form (YUV planes clipped at odd widths)
NEW = (3, 5, 6, 7, 9, 10, 11, 12, 13, 14, 15, 16)
for k in NEW:
    n += len(enc.decompress(rag, scale=(k, 8), all_scales=True))
n += len(enc.decompress_mixed([rag[0], srcs[0]], [dict(scale=(k, 8), all_scales=True) for k in NEW])[0])
for f in ((3, 8), (5, 8), (3, 4), (7, 8), (9, 8), (5, 4), (11, 8), (3, 2), (13, 8), (7, 4), (15, 8), (2, 1)):
    n += len(enc.decompress_yuv(rag, scale=f, all_scales=True))
# CMYK and YCCK sources (cmyk): k_upsample_opts<4> through the one-geometry form, k_upsample_ragged<4> through a mixed
# batch with a 3-component file, at ragged sizes with the 2:1 edge rules
cm = enc.encode_batch(mj.tj3_params(61, 37, subsamp="444", cmyk=True, colorspace=mj._abi.CS_CMYK), np.stack([synth_image(13, 61, 37)[..., [0, 1, 2, 0]]] * 2))
yk = enc.encode_batch(mj.tj3_params(67, 35, subsamp="420", cmyk=True), np.stack([synth_image(14, 67, 35)[..., [0, 1, 2, 1]]] * 2))
for f in (cm, yk):
    n += len(enc.decompress(f, cmyk=True))
    n += len(enc.decompress(f, scale=(1, 2), dct="fast", fancy=False, cmyk=True))
n += len(enc.decompress_mixed([cm[0], yk[0], rag[0]], [dict(cmyk=True), dict(scale=(1, 4), cmyk=True)])[0])
# progressive decode: the default profile (scan search, successive approximation), the standard script with restarts,
# mixed with sequential files, through the coefficient, transcode and pixel routes; then a truncated refinement scan
enc.set_progressive_decode(True)
prog = enc.encode_batch(mj.params_from_switches(["-quality", "75"], w, h), img)
prog_rst = enc.encode_batch(mj.params_from_switches(["-revert", "-progressive", "-restart", "1"], w, h), img)
n += len(enc.read_coefficients(prog + prog_rst + srcs))
n += len(T.transcode(enc, prog, None, ["-rotate", "90"]))
n += len(enc.decompress(prog_rst, scale=(1, 4)))
last = T.parse_source(prog[0]).scans[-1]
try:
    enc.read_coefficients([prog[0][:last.data_offset + last.data_size // 2]])
except mj.B200JpegError as e:
    assert e.code == mj._abi.ERR_BAD_SOURCE, e
enc.set_progressive_decode(False)
print("sanitize cases done:", n, "files, kernel launches", enc.kernel_launches())
enc.close()
