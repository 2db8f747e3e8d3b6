"""The YUV-encoding cases (tj3EncodeYUVPlanes8) shared by tools/make_golden.py --yuv, tests/test_yuv.py and the fuzzer:
the pixel formats and subsamplings of turbojpeg.h, seeded inputs, and a ctypes caller of the reference's
tj3EncodeYUVPlanes8 in oracle/_ref/libturbojpeg_ref.so."""
import ctypes as C
import hashlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
REF_TJ = os.path.join(ROOT, "oracle", "_ref", "libturbojpeg_ref.so")

# TJSAMP_* (turbojpeg.h) in enum order, with the names tj3_params takes
SUBSAMPS = ["444", "422", "420", "gray", "440", "411", "441"]
# TJPF_* in enum order: name -> bytes per pixel (tjPixelSize)
PIXEL_FORMATS = {"RGB": 3, "BGR": 3, "RGBX": 4, "BGRX": 4, "XBGR": 4, "XRGB": 4, "GRAY": 1, "RGBA": 4, "BGRA": 4, "ABGR": 4,
                 "ARGB": 4, "CMYK": 4}
PF_INDEX = {n: i for i, n in enumerate(PIXEL_FORMATS)}
# where R, G, B sit inside a pixel of each RGB-family format (tjRedOffset / tjGreenOffset / tjBlueOffset)
RGB_OFFSETS = {"RGB": (0, 1, 2), "BGR": (2, 1, 0), "RGBX": (0, 1, 2), "BGRX": (2, 1, 0), "XBGR": (3, 2, 1), "XRGB": (1, 2, 3),
               "RGBA": (0, 1, 2), "BGRA": (2, 1, 0), "ABGR": (3, 2, 1), "ARGB": (1, 2, 3)}
TJINIT_COMPRESS, TJPARAM_SUBSAMP = 0, 4


def read_testorig():
    with open(os.path.join(GOLD, "testorig.ppm"), "rb") as f:
        data = f.read()
    parts = data.split(maxsplit=4)
    w, h = int(parts[1]), int(parts[2])
    return np.frombuffer(parts[4][:w * h * 3], np.uint8).reshape(h, w, 3)


def synth_rgb(seed, w, h):
    """Seeded RGB content: smooth gradients (runs of equal chroma) plus noise (every rounding case of the box filters)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * 7 + y * 3) % 256, (x * 2 + y * 11 + 40) % 256, (x * y // 5 + 90) % 256], -1)
    noise = rng.integers(-40, 41, size=(h, w, 3))
    return np.clip(base + noise, 0, 255).astype(np.uint8)


def to_pixel_format(rgb, pf, seed=0):
    """rgb (H, W, 3) -> (H, W, tjPixelSize[pf]) in the layout of TJPF_<pf>; filler / alpha / K samples are seeded noise
    (the conversions must ignore them), GRAY takes the red samples."""
    h, w, _ = rgb.shape
    if pf == "GRAY":
        return np.ascontiguousarray(rgb[..., :1])
    out = np.random.default_rng(seed + 77).integers(0, 256, size=(h, w, PIXEL_FORMATS[pf]), dtype=np.uint8)
    if pf == "CMYK":
        return out
    for c, off in enumerate(RGB_OFFSETS[pf]):
        out[..., off] = rgb[..., c]
    return out


def case_pixels(size, pf):
    """The input of a golden case: size is (w, h) or "testorig"."""
    if size == "testorig":
        rgb = read_testorig()
    else:
        w, h = size
        rgb = synth_rgb(w * 1000 + h, w, h)
    return to_pixel_format(rgb, pf, seed=rgb.shape[0] * 7 + rgb.shape[1])


def md5(a) -> str:
    return hashlib.md5(np.ascontiguousarray(a).tobytes()).hexdigest()


class RefTJ:
    """The reference's TurboJPEG library (oracle/_ref/libturbojpeg_ref.so), called through ctypes."""

    def __init__(self, path=REF_TJ):
        lib = C.CDLL(path)
        lib.tj3Init.argtypes = [C.c_int]; lib.tj3Init.restype = C.c_void_p
        lib.tj3Destroy.argtypes = [C.c_void_p]; lib.tj3Destroy.restype = None
        lib.tj3Set.argtypes = [C.c_void_p, C.c_int, C.c_int]; lib.tj3Set.restype = C.c_int
        lib.tj3GetErrorStr.argtypes = [C.c_void_p]; lib.tj3GetErrorStr.restype = C.c_char_p
        lib.tj3YUVPlaneWidth.argtypes = [C.c_int, C.c_int, C.c_int]; lib.tj3YUVPlaneWidth.restype = C.c_int
        lib.tj3YUVPlaneHeight.argtypes = [C.c_int, C.c_int, C.c_int]; lib.tj3YUVPlaneHeight.restype = C.c_int
        lib.tj3EncodeYUVPlanes8.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]
        lib.tj3EncodeYUVPlanes8.restype = C.c_int
        self.lib = lib
        self.h = lib.tj3Init(TJINIT_COMPRESS)

    def close(self):
        if self.h:
            self.lib.tj3Destroy(self.h)
            self.h = None

    def plane_dims(self, ci, w, h, subsamp):
        s = SUBSAMPS.index(subsamp)
        return self.lib.tj3YUVPlaneWidth(ci, w, s), self.lib.tj3YUVPlaneHeight(ci, h, s)

    def encode_planes(self, pixels, pf, subsamp, pad=0):
        """tj3EncodeYUVPlanes8 of one (H, W, C) image: (list of (ph, pw) planes, None) or (None, the reference's error).
        pad: extra bytes per plane row (strides pw + pad; 0 passes NULL strides)."""
        hgt, w = pixels.shape[:2]
        src = np.ascontiguousarray(pixels)
        self.lib.tj3Set(self.h, TJPARAM_SUBSAMP, SUBSAMPS.index(subsamp))
        nplanes = 1 if subsamp == "gray" else 3
        bufs, dims = [], []
        for ci in range(nplanes):
            pw, ph = self.plane_dims(ci, w, hgt, subsamp)
            dims.append((pw, ph))
            bufs.append(np.zeros((ph, pw + pad), np.uint8))
        ptrs = (C.c_void_p * 3)(*([b.ctypes.data for b in bufs] + [None] * (3 - nplanes)))
        strides = (C.c_int * 3)(*[pw + pad for pw, _ in dims], *([0] * (3 - nplanes))) if pad else None
        rc = self.lib.tj3EncodeYUVPlanes8(self.h, src.ctypes.data, w, 0, hgt, PF_INDEX[pf], ptrs, strides)
        if rc != 0:
            return None, self.lib.tj3GetErrorStr(self.h).decode()
        return [b[:, :pw] for b, (pw, _) in zip(bufs, dims)], None


# the golden matrix: every subsampling x pixel format x size x plane stride (0: NULL strides, 13: pw + 13)
SIZES = [(1, 1), (1, 17), (17, 1), (7, 5), (33, 19), "testorig", (1920, 1080)]
PADS = [0, 13]


def size_id(size):
    return size if isinstance(size, str) else f"{size[0]}x{size[1]}"
