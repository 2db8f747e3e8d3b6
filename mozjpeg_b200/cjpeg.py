"""Host-side mirror of the reference's ``cjpeg`` front end.

``params_from_switches`` turns a cjpeg command line (the switches of
cjpeg.c:315-765 that concern the encode hot path) into a ``b200jpeg_params``
block by making the same API calls, in the same order, as cjpeg's ``main``:

    jpeg_create_compress (profile JCP_MAX_COMPRESSION, jcapimin.c:107-109)
    in_color_space = JCS_RGB ; jpeg_set_defaults            cjpeg.c:860-861
    parse_switches(for_real=FALSE)                          cjpeg.c:869
    <image header: dimensions, colour space>                cjpeg.c:921-928
    jpeg_default_colorspace                                 cjpeg.c:931
    parse_switches(for_real=TRUE)                           cjpeg.c:934
    jpeg_start_compress (optimize_scans off w/o script)     jcapistd.c:53-56

so that the parity tests read like the reference's own bit tests
(CMakeLists.txt:1426-1736: ``cjpeg <switches> testorig.ppm`` -> md5).
All parameter arithmetic happens in libb200jpeg (params.cpp); this file only
sequences the calls.
"""
from __future__ import annotations

import ctypes as C
import re
from typing import List, Sequence, Tuple

from . import _abi as A


class UsageError(ValueError):
    """cjpeg would have printed usage() and exited."""


def _keymatch(arg: str, keyword: str, minchars: int) -> bool:
    """cdjpeg.c keymatch(): case-insensitive prefix match of >= minchars."""
    a = arg.lower()
    if len(a) > len(keyword) or len(a) < minchars:
        return False
    return keyword.startswith(a)


def _set_sample_factors(p: A.Params, arg: str) -> None:
    """rdswitch.c:611-645: listed components, then 1x1 for the rest."""
    parts = arg.split(",") if arg else []
    for ci in range(A.MAX_COMPONENTS):
        if ci < len(parts):
            hv = parts[ci].lower().split("x")
            if len(hv) != 2:
                raise UsageError("can't set sample factors")
            h, v = int(hv[0]), int(hv[1])
            if not (1 <= h <= 4 and 1 <= v <= 4):
                raise UsageError("JPEG sampling factors must be 1..4")
        else:
            h, v = 1, 1
        p.comp_info[ci].h_samp_factor = h
        p.comp_info[ci].v_samp_factor = v


def _text_integers(text: str):
    """rdswitch.c:37-77 read_text_integer over a whole file: ('int', value) / ('sep', char) tokens; '#' starts a
    comment that runs to the end of the line and reads as a newline."""
    out = []
    i, n = 0, len(text)
    while i < n:
        ch = text[i]
        if ch == "#":
            while i < n and text[i] != "\n":
                i += 1
            continue
        if ch.isdigit():
            j = i
            while j < n and text[j].isdigit():
                j += 1
            out.append(("int", int(text[i:j])))
            i = j
            continue
        if not ch.isspace():
            out.append(("sep", ch))
        i += 1
    return out


def _read_quant_tables(p: A.Params, filename: str, force_baseline: bool) -> None:
    """rdswitch.c:83-146: up to NUM_QUANT_TBLS tables of 64 decimal values, each scaled by its slot's q_scale_factor."""
    lib = A.load()
    toks = _text_integers(open(filename).read())
    if any(k != "int" for k, _ in toks):
        raise UsageError(f"Non-numeric data in file {filename}")
    vals = [v for _, v in toks]
    if len(vals) % 64:
        raise UsageError(f"Invalid table data in file {filename}")
    if len(vals) // 64 > A.NUM_QUANT_TBLS:
        raise UsageError(f"Too many tables in file {filename}")
    for t in range(len(vals) // 64):
        tbl = (C.c_uint * 64)(*vals[64 * t:64 * t + 64])
        A.check(lib.b200jpeg_add_quant_table(C.byref(p), t, tbl, p.q_scale_factor[t], int(force_baseline)), "add_quant_table")


def _set_quant_slots(p: A.Params, arg: str) -> None:
    """rdswitch.c:576-612: N[,N,...], the last value replicated over the remaining components."""
    parts = arg.split(",") if arg else []
    val = 0
    for ci in range(A.MAX_COMPONENTS):
        if ci < len(parts):
            try:
                val = int(parts[ci])
            except ValueError:
                raise UsageError("can't set quant slots")
            if not 0 <= val < A.NUM_QUANT_TBLS:
                raise UsageError(f"JPEG quantization tables are numbered 0..{A.NUM_QUANT_TBLS - 1}")
        p.comp_info[ci].quant_tbl_no = val


def _read_scan_script(p: A.Params, filename: str) -> None:
    """rdswitch.c:174-270: entries 'c0 [c1 ..] [: Ss Se Ah Al] ;' - any punctuation other than ':' and ';' is a
    separator.  Validation is left to the library, like jcmaster.c does for the reference."""
    toks = _text_integers(open(filename).read())
    scans = []
    cur: List[int] = []
    prog: List[int] = []
    in_prog = False

    def close():
        nonlocal cur, prog, in_prog
        if not cur:
            raise UsageError(f"Invalid scan entry format in file {filename}")
        if in_prog and len(prog) != 4:
            raise UsageError(f"Invalid scan entry format in file {filename}")
        if len(cur) > 4:
            raise UsageError(f"Too many components in one scan in file {filename}")
        scans.append((cur, prog if in_prog else [0, 63, 0, 0]))
        cur, prog, in_prog = [], [], False

    for kind, v in toks:
        if kind == "int":
            (prog if in_prog else cur).append(v)
        elif v == ":":
            if in_prog or not cur:
                raise UsageError(f"Invalid scan entry format in file {filename}")
            in_prog = True
        elif v == ";":
            close()
    if cur or in_prog:
        close()                                               # the last entry may end at EOF
    if len(scans) > 64:
        raise UsageError(f"Too many scans defined in file {filename}")
    if scans:
        p.num_scans = len(scans)
        for i, (comps, pr) in enumerate(scans):
            si = p.scan_info[i]
            si.comps_in_scan = len(comps)
            for k in range(4):
                si.component_index[k] = comps[k] if k < len(comps) else 0
            si.Ss, si.Se, si.Ah, si.Al = pr
        p.optimize_scans = 0                                  # rdswitch.c:262-263


def _parse(p: A.Params, argv: Sequence[str], for_real: bool) -> None:
    lib = A.load()
    force_baseline = False
    simple_progressive = p.num_scans != 0          # cjpeg.c:343
    qualityarg = samplearg = qtablefile = qslotsarg = scansarg = None
    psv, pt = 0, 0
    i = 0
    n = len(argv)

    def nextarg(what: str) -> str:
        nonlocal i
        i += 1
        if i >= n:
            raise UsageError(f"missing argument for {what}")
        return argv[i]

    while i < n:
        arg = argv[i]
        if not arg.startswith("-"):
            raise UsageError(f"unexpected file argument {arg!r}")
        a = arg[1:]
        if _keymatch(a, "baseline", 1):
            force_baseline = True
            simple_progressive = False
            p.num_scans = 0
        elif _keymatch(a, "dct", 2):
            v = nextarg("dct")
            if _keymatch(v, "int", 1): p.dct_method = A.DCT_ISLOW
            elif _keymatch(v, "fast", 2): p.dct_method = A.DCT_IFAST
            elif _keymatch(v, "float", 2): p.dct_method = A.DCT_FLOAT
            else: raise UsageError("invalid argument for dct")
        elif _keymatch(a, "fastcrush", 4):
            p.optimize_scans = 0
        elif _keymatch(a, "grayscale", 2) or _keymatch(a, "greyscale", 2):
            A.check(lib.b200jpeg_set_colorspace(C.byref(p), A.CS_GRAYSCALE), "set_colorspace")
        elif _keymatch(a, "rgb", 3):
            A.check(lib.b200jpeg_set_colorspace(C.byref(p), A.CS_RGB), "set_colorspace")
        elif _keymatch(a, "lossless", 1):
            # cjpeg.c:459-480: "psv[,Pt]"; executed after the other switches, once data_precision is known
            v = nextarg("lossless")
            m = re.match(r"\s*([+-]?\d+)(.?)", v)
            if not m or (m.group(2) and m.group(2) != ","):
                raise UsageError("invalid argument for lossless")
            psv = int(m.group(1))
            rest = v.split(",", 1)
            if len(rest) == 2:
                m2 = re.match(r"\s*([+-]?\d+)", rest[1])
                if m2:
                    pt = int(m2.group(1))
        elif _keymatch(a, "lambda1", 7):
            p.lambda_log_scale1 = float(nextarg("lambda1"))
        elif _keymatch(a, "lambda2", 7):
            p.lambda_log_scale2 = float(nextarg("lambda2"))
        elif _keymatch(a, "dc-scan-opt", 3):
            p.dc_scan_opt_mode = int(nextarg("dc-scan-opt"))
        elif _keymatch(a, "optimize", 1) or _keymatch(a, "optimise", 1):
            p.optimize_coding = 1
        elif _keymatch(a, "precision", 3):
            v = nextarg("precision")
            if int(v) not in (8, 12, 16):
                raise UsageError("precision must be 8, 12 or 16")
            p.data_precision = int(v)
        elif _keymatch(a, "progressive", 1):
            simple_progressive = True
        elif _keymatch(a, "quality", 1):
            qualityarg = nextarg("quality")
        elif _keymatch(a, "qslots", 2):
            qslotsarg = nextarg("qslots")
        elif _keymatch(a, "qtables", 2):
            qtablefile = nextarg("qtables")
        elif _keymatch(a, "scans", 2):
            scansarg = nextarg("scans")
        elif _keymatch(a, "quant-table", 7):
            v = int(nextarg("quant-table"))
            if not 0 <= v <= 8:
                raise UsageError(f"{v} is invalid argument for quant-table")
            p.quant_tbl_master_idx = v                       # jcext.c JINT_BASE_QUANT_TBL_IDX
            lib.b200jpeg_set_quality(C.byref(p), 75, 1)      # cjpeg.c:595
        elif _keymatch(a, "quant-baseline", 7):
            force_baseline = True
        elif _keymatch(a, "restart", 1):
            v = nextarg("restart")
            if v[-1:] in "bB":
                p.restart_interval = int(v[:-1]); p.restart_in_rows = 0
            else:
                p.restart_in_rows = int(v)
        elif _keymatch(a, "revert", 3):
            w, h = p.image_width, p.image_height
            lib.b200jpeg_set_defaults(C.byref(p), A.PROFILE_FASTEST)   # cjpeg.c:623-626
            p.image_width, p.image_height = w, h
        elif _keymatch(a, "sample", 2):
            samplearg = nextarg("sample")
        elif _keymatch(a, "smooth", 2):
            p.smoothing_factor = int(nextarg("smooth"))
        elif _keymatch(a, "notrellis-dc", 11):
            p.trellis_quant_dc = 0
        elif _keymatch(a, "notrellis", 1):
            p.trellis_quant = 0
        elif _keymatch(a, "trellis-dc-ver-weight", 11):          # cjpeg.c:667-672
            p.trellis_delta_dc_weight = float(nextarg("trellis-dc-ver-weight"))
        elif _keymatch(a, "trellis-dc", 9):
            p.trellis_quant_dc = 1
        elif _keymatch(a, "tune-psnr", 6):
            p.quant_tbl_master_idx = 1; p.lambda_log_scale1 = 9.0; p.lambda_log_scale2 = 0.0; p.use_lambda_weight_tbl = 0
            lib.b200jpeg_set_quality(C.byref(p), 75, 1)
        elif _keymatch(a, "tune-ssim", 6):
            p.quant_tbl_master_idx = 1; p.lambda_log_scale1 = 11.5; p.lambda_log_scale2 = 12.75; p.use_lambda_weight_tbl = 0
            lib.b200jpeg_set_quality(C.byref(p), 75, 1)
        elif _keymatch(a, "tune-ms-ssim", 6):
            p.quant_tbl_master_idx = 3; p.lambda_log_scale1 = 12.0; p.lambda_log_scale2 = 13.0; p.use_lambda_weight_tbl = 1
            lib.b200jpeg_set_quality(C.byref(p), 75, 1)
        elif _keymatch(a, "tune-hvs-psnr", 6):
            p.quant_tbl_master_idx = 3; p.lambda_log_scale1 = 14.75; p.lambda_log_scale2 = 16.5; p.use_lambda_weight_tbl = 1
            lib.b200jpeg_set_quality(C.byref(p), 75, 1)
        elif _keymatch(a, "noovershoot", 11):
            p.overshoot_deringing = 0
        elif _keymatch(a, "nojfif", 6):
            p.write_JFIF_header = 0
        else:
            raise UsageError(f"unknown or out-of-scope option {arg!r}")
        i += 1

    if for_real:
        if qualityarg is not None:
            # rdswitch.c:524-573 set_quality_ratings
            vals = qualityarg.split(",")
            val = 75.0
            for t in range(A.NUM_QUANT_TBLS):
                if t < len(vals):
                    val = float(vals[t])
                p.q_scale_factor[t] = int(lib.b200jpeg_float_quality_scaling(val))
            lib.b200jpeg_default_qtables(C.byref(p), int(force_baseline))
            if val >= 90:
                _set_sample_factors(p, "1x1")
            elif val >= 80:
                _set_sample_factors(p, "2x1")
        if qtablefile is not None:
            _read_quant_tables(p, qtablefile, force_baseline)
        if qslotsarg is not None:
            _set_quant_slots(p, qslotsarg)
        if samplearg is not None:
            _set_sample_factors(p, samplearg)
        if simple_progressive:
            A.check(lib.b200jpeg_simple_progression(C.byref(p)), "simple_progression")
        if psv != 0:                                                  # cjpeg.c:752-755
            A.check(lib.b200jpeg_enable_lossless(C.byref(p), psv, pt), "enable_lossless")
        if scansarg is not None:
            _read_scan_script(p, scansarg)


def params_from_switches(switches: Sequence[str], width: int, height: int,
                         input_components: int = 3, in_color_space: int = None,
                         jpeg_color_space: int = None) -> A.Params:
    """What cjpeg's cinfo looks like at jpeg_start_compress for ``switches``.

    ``in_color_space`` (default: grayscale for 1 component, else RGB) is what the image header reports, e.g.
    CS_CMYK for a 4-sample CMYK source; ``jpeg_color_space`` is a jpeg_set_colorspace call made right after
    jpeg_default_colorspace, before the switches are applied for real."""
    lib = A.load()
    p = A.Params()
    p.in_color_space = A.CS_RGB
    p.input_components = 3
    p.data_precision = 8
    lib.b200jpeg_set_defaults(C.byref(p), A.PROFILE_MAX_COMPRESSION)
    _parse(p, list(switches), False)
    # image header (rdppm.c start_input_ppm): P5 -> grayscale, P6 -> RGB
    if in_color_space is None:
        in_color_space = A.CS_GRAYSCALE if input_components == 1 else A.CS_RGB
    p.in_color_space = in_color_space
    p.input_components = input_components
    p.image_width, p.image_height = width, height
    A.check(lib.b200jpeg_default_colorspace(C.byref(p)), "default_colorspace")
    if jpeg_color_space is not None:
        A.check(lib.b200jpeg_set_colorspace(C.byref(p), jpeg_color_space), "set_colorspace")
    _parse(p, list(switches), True)
    # jpeg_start_compress (jcapistd.c:53-56)
    if p.num_scans == 0:
        p.optimize_scans = 0
    return p


def read_pnm(data: bytes):
    """Minimal binary PGM/PPM reader (P5/P6) -> (w, h, ncomp, maxval, samples): samples is an (h, w, ncomp) uint8 array
    for maxval <= 255, else uint16 (two bytes per sample, big-endian in the file, as rdppm.c reads them)."""
    import numpy as np
    toks: List[bytes] = []
    pos = 0
    while len(toks) < 4:
        while data[pos:pos + 1].isspace():
            pos += 1
        if data[pos:pos + 1] == b"#":
            while data[pos:pos + 1] not in (b"\n", b""):
                pos += 1
            continue
        st = pos
        while not data[pos:pos + 1].isspace():
            pos += 1
        toks.append(data[st:pos])
    pos += 1
    magic, w, h, maxv = toks[0], int(toks[1]), int(toks[2]), int(toks[3])
    if magic not in (b"P5", b"P6") or not 1 <= maxv <= 65535:
        raise ValueError("only binary PGM/PPM (P5/P6) supported")
    nc = 3 if magic == b"P6" else 1
    if maxv <= 255:
        a = np.frombuffer(data[pos:pos + w * h * nc], dtype=np.uint8)
    else:
        a = np.frombuffer(data[pos:pos + 2 * w * h * nc], dtype=">u2").astype(np.uint16)
    if a.size != w * h * nc:
        raise ValueError("PGM/PPM file is truncated")
    return w, h, nc, maxv, a.reshape(h, w, nc)


def pnm_samples(maxval: int, samples, data_precision: int):
    """The samples as the encoder takes them at ``data_precision``.  rdppm.c rescales every maxval other than the
    precision's largest sample value (its rescale[] tables); that is not mirrored here, so such a file is refused rather
    than coded with samples the reference would not see."""
    if maxval != (1 << data_precision) - 1:
        raise ValueError(f"maxval {maxval} at data precision {data_precision}: only maxval {(1 << data_precision) - 1} "
                         "is read without rescaling")
    return samples


def read_ppm(data: bytes) -> Tuple[int, int, int, bytes]:
    """Minimal binary PGM/PPM reader (P5/P6, maxval 255) -> (w, h, ncomp, samples)."""
    w, h, nc, maxv, a = read_pnm(data)
    if maxv != 255:
        raise ValueError("only binary 8-bit PGM/PPM supported")
    return w, h, nc, a.tobytes()


def main(argv: Sequence[str] = None) -> int:
    """``python -m mozjpeg_b200.cjpeg [switches] [-outfile name] file.ppm [more.ppm ...]`` - cjpeg's command line on
    the device path.  Several input files of one size are encoded as one batch (outputs: <input>.jpg)."""
    import sys
    import numpy as np
    from . import Encoder
    args = list(sys.argv[1:] if argv is None else argv)
    outfile = None
    switches: List[str] = []
    files: List[str] = []
    takes_arg = ("dct", "lambda1", "lambda2", "dc-scan-opt", "lossless", "precision", "quality", "qslots", "qtables", "scans", "quant-table",
                 "restart", "sample", "smooth", "trellis-dc-ver-weight")
    i = 0
    while i < len(args):
        a = args[i]
        if a.startswith("-") and len(a) > 1:
            if _keymatch(a[1:], "outfile", 4):
                outfile = args[i + 1]; i += 2; continue
            switches.append(a)
            if any(_keymatch(a[1:], k, 2 if k not in ("quality", "restart") else 1) for k in takes_arg) and not _keymatch(a[1:], "quant-baseline", 7):
                switches.append(args[i + 1]); i += 1
        else:
            files.append(a)
        i += 1
    if not files:
        print("usage: python -m mozjpeg_b200.cjpeg [switches] [-outfile name] file.ppm [more.ppm ...]", file=sys.stderr)
        return 2
    raw = []
    for f in files:
        w, h, nc, maxv, a = read_pnm(open(f, "rb").read())
        raw.append((maxv, a))
    if len({a.shape for _, a in raw}) != 1:
        print("all input files of one call must have the same size", file=sys.stderr)
        return 2
    h, w, nc = raw[0][1].shape
    p = params_from_switches(switches, w, h, nc)
    try:
        imgs = [pnm_samples(maxv, a, p.data_precision) for maxv, a in raw]
    except ValueError as e:
        print(str(e), file=sys.stderr)
        return 2
    out = Encoder(0).encode_batch(p, np.stack(imgs))
    for f, jpg in zip(files, out):
        name = outfile if (outfile and len(files) == 1) else f.rsplit(".", 1)[0] + ".jpg"
        with open(name, "wb") as fo:
            fo.write(jpg)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
