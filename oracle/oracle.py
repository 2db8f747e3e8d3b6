"""TEST INFRASTRUCTURE -- ctypes access to the two CPU checkers.

* ``liboracle.so``      : our plain-C restatement (oracle/jpeg_oracle.c)
* ``_ref/librefshim.so``: a thin driver around the UNMODIFIED reference
  library compiled from /root/reference by oracle/Makefile (travels to the GPU
  box as a prebuilt, git-ignored file).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs may import this module.  The product
(mozjpeg_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)



def _sibling(name):
    """mozjpeg_b200/<name>.py (pure Python: the parameter block's ctypes layout, the synthetic-image generator).  With
    B200JPEG_ORACLE_STANDALONE=1 (bench.py's reference arm) the file is loaded by path, so that the process never
    imports the package and therefore never maps libb200jpeg.so."""
    if os.environ.get("B200JPEG_ORACLE_STANDALONE") == "1" and "mozjpeg_b200" not in sys.modules:
        import importlib.util
        spec = importlib.util.spec_from_file_location("_b200_standalone_" + name, os.path.join(_ROOT, "mozjpeg_b200", name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    import importlib
    return importlib.import_module("mozjpeg_b200." + name)


A = _sibling("_abi")  # data layout of b200jpeg_params only


def build(quiet: bool = True) -> None:
    """Compile liboracle.so and, when /root/reference is present, oracle/_ref/."""
    r = subprocess.run(["make", "-C", _HERE, "-j8", "all"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + r.stdout[-3000:] + r.stderr[-3000:])


class OrcDebug(C.Structure):
    _fields_ = [
        ("ncomp", C.c_int), ("wib", C.c_int * 4), ("hib", C.c_int * 4), ("wpad", C.c_int * 4), ("hpad", C.c_int * 4),
        ("plain", C.POINTER(C.c_int16) * 4), ("raw", C.POINTER(C.c_int16) * 4), ("final_", C.POINTER(C.c_int16) * 4),
        ("trellis_dc", A.HuffTbl * 4), ("trellis_ac", A.HuffTbl * 4),
        ("nscans", C.c_int),
        ("scan_dc", (A.HuffTbl * 4) * A.MAX_SCANS), ("scan_ac", (A.HuffTbl * 4) * A.MAX_SCANS),
        ("scan_bytes", C.c_size_t * A.MAX_SCANS),
    ]


_orc = None


def orc() -> C.CDLL:
    global _orc
    if _orc is None:
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            build()
        lib = C.CDLL(path)
        lib.orc_encode.argtypes = [C.POINTER(A.Params), C.c_void_p, C.c_size_t, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t), C.POINTER(OrcDebug)]
        lib.orc_encode.restype = C.c_int
        lib.orc_free.argtypes = [C.c_void_p]
        lib.orc_debug_free.argtypes = [C.POINTER(OrcDebug)]
        lib.orc_fdct_islow.argtypes = [C.POINTER(C.c_int)]
        lib.orc_deringing.argtypes = [C.POINTER(C.c_int), C.c_int]
        lib.orc_gen_optimal_table.argtypes = [C.POINTER(C.c_long), C.POINTER(A.HuffTbl)]
        _orc = lib
    return _orc


class OracleResult:
    def __init__(self, jpeg: bytes, dbg: Optional[dict]):
        self.jpeg = jpeg
        self.dbg = dbg


def oracle_encode(p: A.Params, pixels: np.ndarray, want_debug: bool = False) -> OracleResult:
    """Run the C restatement on an (H, W, C) or (H, W) uint8 array (uint16 for 12-bit precision)."""
    lib = orc()
    pix = np.ascontiguousarray(pixels, dtype=np.uint16 if p.data_precision == 12 else np.uint8)
    pitch = pix.strides[0]
    out = C.POINTER(C.c_uint8)()
    n = C.c_size_t(0)
    dbg = OrcDebug()
    rc = lib.orc_encode(C.byref(p), pix.ctypes.data, pitch, C.byref(out), C.byref(n), C.byref(dbg) if want_debug else None)
    if rc != 0:
        raise RuntimeError(f"oracle encode failed: {rc}")
    data = C.string_at(out, n.value)
    lib.orc_free(out)
    d = None
    if want_debug:
        d = {"ncomp": dbg.ncomp, "wib": list(dbg.wib), "hib": list(dbg.hib), "wpad": list(dbg.wpad), "hpad": list(dbg.hpad),
             "plain": [], "raw": [], "final": [], "nscans": dbg.nscans, "scan_bytes": list(dbg.scan_bytes)[:dbg.nscans]}
        for ci in range(dbg.ncomp):
            cnt = dbg.wpad[ci] * dbg.hpad[ci] * 64
            shape = (dbg.hpad[ci], dbg.wpad[ci], 64)
            for key, ptr in (("plain", dbg.plain[ci]), ("raw", dbg.raw[ci]), ("final", dbg.final_[ci])):
                d[key].append(np.ctypeslib.as_array(ptr, shape=(cnt,)).copy().reshape(shape))
        d["trellis_dc"] = [_huff_to_py(dbg.trellis_dc[i]) for i in range(dbg.ncomp)]
        d["trellis_ac"] = [_huff_to_py(dbg.trellis_ac[i]) for i in range(dbg.ncomp)]
        d["scan_dc"] = [[_huff_to_py(dbg.scan_dc[s][k]) for k in range(4)] for s in range(dbg.nscans)]
        d["scan_ac"] = [[_huff_to_py(dbg.scan_ac[s][k]) for k in range(4)] for s in range(dbg.nscans)]
        lib.orc_debug_free(C.byref(dbg))
    return OracleResult(data, d)


def _huff_to_py(h: A.HuffTbl) -> Tuple[Tuple[int, ...], Tuple[int, ...]]:
    bits = tuple(h.bits)
    n = sum(bits[1:])
    return bits, tuple(h.huffval)[:n]


# ---------------------------------------------------------------------------
# the real reference (oracle/_ref)
# ---------------------------------------------------------------------------
class RefCfg(C.Structure):
    _fields_ = [
        ("revert", C.c_int), ("baseline", C.c_int), ("has_quality", C.c_int), ("quality", C.c_float),
        ("samp_h", C.c_int * 4), ("samp_v", C.c_int * 4),
        ("optimize", C.c_int), ("progressive", C.c_int), ("fastcrush", C.c_int), ("notrellis", C.c_int),
        ("trellis_dc", C.c_int), ("noovershoot", C.c_int), ("dct", C.c_int),
        ("restart", C.c_int), ("restart_blocks", C.c_int), ("grayscale", C.c_int), ("quant_table", C.c_int),
        ("precision", C.c_int), ("has_lambda1", C.c_int), ("has_lambda2", C.c_int),
        ("lambda1", C.c_float), ("lambda2", C.c_float), ("tjapi", C.c_int), ("input_gray", C.c_int),
        ("ext_use_scans_in_trellis", C.c_int), ("ext_trellis_freq_split", C.c_int), ("ext_trellis_eob_opt", C.c_int),
        ("ext_trellis_q_opt", C.c_int), ("ext_trellis_num_loops", C.c_int),
        ("has_dc_ver_weight", C.c_int), ("dc_ver_weight", C.c_float),
    ]


REF_DIR = os.path.join(_HERE, "_ref")
_ref = None


def ref_available() -> bool:
    return os.path.exists(os.path.join(REF_DIR, "librefshim.so"))


def ref() -> C.CDLL:
    global _ref
    if _ref is None:
        if not ref_available():
            build()
        if not ref_available():
            raise RuntimeError("oracle/_ref is not built and /root/reference is absent")
        lib = C.CDLL(os.path.join(REF_DIR, "librefshim.so"))
        lib.refshim_encode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(RefCfg), C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_ulong), C.c_char_p, C.c_int]
        lib.refshim_encode.restype = C.c_int
        lib.refshim_free.argtypes = [C.c_void_p]
        lib.refshim_read_coefs.argtypes = [C.c_char_p, C.c_ulong, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_uint16), C.POINTER(C.POINTER(C.c_int16))]
        lib.refshim_read_coefs.restype = C.c_int
        lib.refshim_fdct_islow.argtypes = [C.POINTER(C.c_int)]
        _ref = lib
    return _ref


def refcfg_from_switches(switches: Sequence[str], input_gray: bool = False) -> RefCfg:
    """The subset of cjpeg switches the shim understands (canonical order:
    the shim applies them in a fixed order, so tests pass them that way too)."""
    c = RefCfg()
    c.trellis_dc = -1; c.dct = -1; c.quant_table = -1; c.precision = 8
    c.ext_use_scans_in_trellis = c.ext_trellis_freq_split = c.ext_trellis_eob_opt = c.ext_trellis_q_opt = c.ext_trellis_num_loops = -1
    c.input_gray = int(input_gray)
    it = iter(switches)
    for s in it:
        if s == "-revert": c.revert = 1
        elif s == "-baseline": c.baseline = 1
        elif s == "-quality": c.has_quality = 1; c.quality = float(next(it))
        elif s == "-sample":
            parts = next(it).split(",")
            for i, hv in enumerate(parts[:4]):
                h, v = hv.lower().split("x"); c.samp_h[i] = int(h); c.samp_v[i] = int(v)
        elif s == "-optimize": c.optimize = 1
        elif s == "-progressive": c.progressive = 1
        elif s == "-fastcrush": c.fastcrush = 1
        elif s == "-notrellis": c.notrellis = 1
        elif s == "-notrellis-dc": c.trellis_dc = 0
        elif s == "-trellis-dc": c.trellis_dc = 1
        elif s == "-noovershoot": c.noovershoot = 1
        elif s == "-dct": c.dct = {"int": 0, "fast": 1, "float": 2}[next(it)]
        elif s == "-restart":
            v = next(it)
            if v[-1] in "bB": c.restart = int(v[:-1]); c.restart_blocks = 1
            else: c.restart = int(v)
        elif s == "-grayscale": c.grayscale = 1
        elif s == "-precision": c.precision = int(next(it))
        elif s == "-quant-table": c.quant_table = int(next(it))
        elif s == "-trellis-dc-ver-weight": c.has_dc_ver_weight = 1; c.dc_ver_weight = float(next(it))
        elif s == "-lambda1": c.has_lambda1 = 1; c.lambda1 = float(next(it))
        elif s == "-lambda2": c.has_lambda2 = 1; c.lambda2 = float(next(it))
        else: raise ValueError(f"refshim: unsupported switch {s}")
    return c


def ref_encode(pixels: np.ndarray, switches: Sequence[str], ext: Optional[dict] = None) -> bytes:
    """Encode with the UNMODIFIED reference (libjpeg API, cjpeg switch semantics).  ext: extension parameters cjpeg has
    no switch for, e.g. {"use_scans_in_trellis": 1, "trellis_freq_split": 8} (set through jpeg_c_set_*_param)."""
    lib = ref()
    gray = pixels.ndim == 2 or pixels.shape[2] == 1
    try:
        cfg = refcfg_from_switches(switches, gray)
    except ValueError:
        if ext:
            raise
        return _ref_cjpeg_pixels(pixels, switches)      # a switch only the reference's own cjpeg parses (8-bit input)
    for k, v in (ext or {}).items():
        setattr(cfg, "ext_" + k, int(v))
    pix = np.ascontiguousarray(pixels, dtype=np.uint16 if cfg.precision == 12 else np.uint8)
    out = C.POINTER(C.c_uint8)(); n = C.c_ulong(0)
    err = C.create_string_buffer(256)
    rc = lib.refshim_encode(pix.ctypes.data, pix.shape[1], pix.shape[0], pix.strides[0] // pix.itemsize, C.byref(cfg), C.byref(out), C.byref(n), err, 256)
    if rc != 0:
        raise RuntimeError("reference encode failed: " + err.value.decode())
    data = C.string_at(out, n.value)
    lib.refshim_free(out)
    return data


def _plane_args(planes):
    arrs = [np.ascontiguousarray(a, dtype=np.uint8) for a in planes]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    return arrs, ptrs


def oracle_encode_raw(p: A.Params, planes) -> bytes:
    """C restatement on raw-data input: planes[ci] = (hib*8, wib*8) uint8 (jpeg_write_raw_data semantics)."""
    lib = orc()
    lib.orc_encode_raw.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]
    lib.orc_encode_raw.restype = C.c_int
    arrs, ptrs = _plane_args(planes)
    pitch = (C.c_size_t * len(arrs))(*[a.strides[0] for a in arrs])
    out = C.POINTER(C.c_uint8)(); n = C.c_size_t(0)
    rc = lib.orc_encode_raw(C.byref(p), ptrs, pitch, C.byref(out), C.byref(n))
    if rc != 0:
        raise RuntimeError(f"oracle raw encode failed: {rc}")
    data = C.string_at(out, n.value)
    lib.orc_free(out)
    return data


def ref_encode_raw(planes, width: int, height: int, switches: Sequence[str]) -> bytes:
    """The UNMODIFIED reference through jpeg_write_raw_data."""
    lib = ref()
    lib.refshim_encode_raw.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_ulong), C.c_char_p, C.c_int]
    lib.refshim_encode_raw.restype = C.c_int
    arrs, ptrs = _plane_args(planes)
    pitch = (C.c_int * len(arrs))(*[a.strides[0] for a in arrs])
    cfg = refcfg_from_switches(switches, len(arrs) == 1)
    out = C.POINTER(C.c_uint8)(); n = C.c_ulong(0)
    err = C.create_string_buffer(256)
    rc = lib.refshim_encode_raw(ptrs, pitch, width, height, len(arrs), C.byref(cfg), C.byref(out), C.byref(n), err, 256)
    if rc != 0:
        raise RuntimeError("reference raw encode failed: " + err.value.decode())
    data = C.string_at(out, n.value)
    lib.refshim_free(out)
    return data


def ref_read_coefs(jpeg: bytes) -> Dict[str, object]:
    """jpeg_read_coefficients via the reference decoder: per-component
    [hib][wib][64] int16 (natural order) + quant tables."""
    lib = ref()
    nc = C.c_int(0); wib = (C.c_int * 4)(); hib = (C.c_int * 4)(); qt = (C.c_uint16 * 256)()
    rc = lib.refshim_read_coefs(jpeg, len(jpeg), C.byref(nc), wib, hib, qt, None)
    if rc != 0:
        raise RuntimeError("reference decode failed")
    arrs = [np.zeros((hib[i], wib[i], 64), dtype=np.int16) for i in range(nc.value)]
    ptrs = (C.POINTER(C.c_int16) * 4)()
    for i, a in enumerate(arrs):
        ptrs[i] = a.ctypes.data_as(C.POINTER(C.c_int16))
    rc = lib.refshim_read_coefs(jpeg, len(jpeg), C.byref(nc), wib, hib, qt, ptrs)
    if rc != 0:
        raise RuntimeError("reference decode failed")
    return {"coefs": arrs, "qt": np.array(qt, dtype=np.uint16).reshape(4, 64)[:nc.value]}


_refshim_tree = None


def ref_read_coefs_warn(jpeg: bytes):
    """jpeg_read_coefficients via the reference decoder, with its warnings counted: (planes or None where the
    reference stops with an error, warnings emitted).  Runs build/librefshim.so, which build() compiles from this
    tree's refshim.c against the reference library (oracle/_ref/ can hold a driver built from an older refshim.c)."""
    global _refshim_tree
    if _refshim_tree is None:
        path = os.path.join(_ROOT, "build", "librefshim.so")
        if not os.path.exists(path):
            raise RuntimeError("build/librefshim.so is missing: run build() where oracle/_ref is built")
        _refshim_tree = C.CDLL(path)
    fn = _refshim_tree.refshim_read_coefs_warn
    fn.argtypes = [C.c_char_p, C.c_ulong, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_uint16),
                   C.POINTER(C.POINTER(C.c_int16)), C.POINTER(C.c_int)]
    fn.restype = C.c_int
    nc = C.c_int(0); wib = (C.c_int * 4)(); hib = (C.c_int * 4)(); warn = C.c_int(0)
    if fn(jpeg, len(jpeg), C.byref(nc), wib, hib, None, None, C.byref(warn)) != 0:
        return None, warn.value
    arrs = [np.zeros((hib[i], wib[i], 64), dtype=np.int16) for i in range(nc.value)]
    ptrs = (C.POINTER(C.c_int16) * 4)()
    for i, a in enumerate(arrs):
        ptrs[i] = a.ctypes.data_as(C.POINTER(C.c_int16))
    if fn(jpeg, len(jpeg), C.byref(nc), wib, hib, None, ptrs, C.byref(warn)) != 0:
        return None, warn.value
    return arrs, warn.value


def _ref_cjpeg_pixels(pixels: np.ndarray, switches: Sequence[str]) -> bytes:
    """The reference's cjpeg binary on an in-memory 8-bit image (written out as a PGM/PPM first)."""
    import tempfile
    pix = np.ascontiguousarray(pixels, dtype=np.uint8)
    gray = pix.ndim == 2 or pix.shape[2] == 1
    with tempfile.NamedTemporaryFile(suffix=".pgm" if gray else ".ppm") as f:
        f.write(b"%s\n%d %d\n255\n" % (b"P5" if gray else b"P6", pix.shape[1], pix.shape[0])); f.write(pix.tobytes()); f.flush()
        return ref_cjpeg(f.name, switches)


def ref_cjpeg(ppm_path: str, switches: Sequence[str]) -> bytes:
    """Run the reference's own cjpeg binary (oracle/_ref/cjpeg)."""
    exe = os.path.join(REF_DIR, "cjpeg")
    r = subprocess.run([exe, *switches, ppm_path], capture_output=True)
    if r.returncode != 0:
        raise RuntimeError("cjpeg failed: " + r.stderr.decode())
    return r.stdout


synth_image = _sibling("synth").synth_image  # input generator shared with bench.py
synth_image12 = _sibling("synth").synth_image12


def oracle_encode_coefs(p: A.Params, planes) -> bytes:
    """C restatement on coefficient input: planes[ci] = (hib, wib, 64) int16, natural order (jpeg_write_coefficients)."""
    lib = orc()
    lib.orc_encode_coefs.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]
    lib.orc_encode_coefs.restype = C.c_int
    arrs = [np.ascontiguousarray(a, dtype=np.int16) for a in planes]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    pitch = (C.c_size_t * len(arrs))(*[a.strides[0] // 128 for a in arrs])
    out = C.POINTER(C.c_uint8)(); n = C.c_size_t(0)
    rc = lib.orc_encode_coefs(C.byref(p), ptrs, pitch, C.byref(out), C.byref(n))
    if rc != 0:
        raise RuntimeError(f"oracle coefficient encode failed: {rc}")
    data = C.string_at(out, n.value)
    lib.orc_free(out)
    return data


def ref_jpegtran(jpeg: bytes, switches: Sequence[str]) -> bytes:
    """The reference's own jpegtran binary (oracle/_ref/jpegtran) on an in-memory file."""
    exe = os.path.join(REF_DIR, "jpegtran")
    r = subprocess.run([exe, *switches], input=jpeg, capture_output=True)
    if r.returncode != 0:
        raise RuntimeError("jpegtran failed: " + r.stderr.decode())
    return r.stdout
