"""``python -m mozjpeg_b200.djpeg`` -- the reference's djpeg command line on the device path, for the switches that set
decompress options (djpeg.c parse_switches, with its abbreviations) and PPM / PGM output framed as wrppm.c writes it:

  -scale M/N            scale_num / scale_denom (the block sizes 1, 2, 4 and 8: 1/8, 1/4, 1/2, 1/1, and fractions that
                        fall into them)
  -dct int|fast|float   dct_method
  -nosmooth             do_fancy_upsampling = FALSE
  -fast                 JDCT_IFAST and no fancy upsampling (the quantization settings it also makes need -colors)
  -grayscale, -rgb      out_color_space
  -pnm / -ppm           the output format (the default)
  -outfile name

Every other output format or option (-bmp, -gif, -targa, -colors, -dither, -crop, -skip, -rgb565, ...) exits with 1
and says it is not on the device path."""
from typing import List, Sequence

import numpy as np


class NotOnDevice(Exception):
    pass


def _keymatch(arg: str, keyword: str, minchars: int) -> bool:
    """cdjpeg.c keymatch: arg is a prefix of keyword of at least minchars characters"""
    return minchars <= len(arg) <= len(keyword) and keyword.startswith(arg)


def parse(switches: Sequence[str]) -> dict:
    """djpeg switches -> the keyword options of Encoder.decompress (scale, dct, fancy, colorspace)"""
    o = dict(scale=(1, 1), dct="int", fancy=True, colorspace=None)
    i = 0
    sw = list(switches)
    while i < len(sw):
        a = sw[i]
        k = a[1:] if a.startswith("-") else a

        def value():
            if i + 1 >= len(sw):
                raise ValueError(f"missing argument for {a}")
            return sw[i + 1]
        if _keymatch(k, "scale", 1):
            v = value(); i += 1
            try:
                num, denom = (int(t) for t in v.split("/"))
            except ValueError:
                raise ValueError(f"bad -scale argument {v!r}") from None
            o["scale"] = (num, denom)
        elif _keymatch(k, "dct", 2):
            v = value(); i += 1
            for name in ("int", "fast", "float"):
                if _keymatch(v, name, 2):
                    o["dct"] = name
                    break
            else:
                raise ValueError(f"bad -dct argument {v!r}")
        elif _keymatch(k, "nosmooth", 3):
            o["fancy"] = False
        elif _keymatch(k, "fast", 1):
            o["dct"] = "fast"; o["fancy"] = False
        elif _keymatch(k, "grayscale", 2) or _keymatch(k, "greyscale", 2):
            o["colorspace"] = "gray"
        elif _keymatch(k, "rgb565", 4):
            raise NotOnDevice(f"{a}: RGB565 output is not on the device path")
        elif _keymatch(k, "rgb", 2):
            o["colorspace"] = "rgb"
        elif _keymatch(k, "ppm", 1) or _keymatch(k, "pnm", 1):
            pass
        else:
            raise NotOnDevice(f"{a}: this output format or option is not on the device path")
        i += 1
    return o


def ppm_bytes(px: np.ndarray) -> bytes:
    """wrppm.c's file for 8-bit samples: P5 for one component, P6 for RGB, then the rows"""
    px = np.ascontiguousarray(px, dtype=np.uint8)
    h, w = px.shape[:2]
    magic = "P5" if px.ndim == 2 or px.shape[2] == 1 else "P6"
    return f"{magic}\n{w} {h}\n255\n".encode() + px.tobytes()


def main(argv: Sequence[str] = None) -> int:
    """``python -m mozjpeg_b200.djpeg [switches] [-outfile name] file.jpg``"""
    import sys
    from . import Encoder
    args = list(sys.argv[1:] if argv is None else argv)
    outfile = None
    switches: List[str] = []
    files: List[str] = []
    i = 0
    while i < len(args):
        a = args[i]
        if a.startswith("-") and len(a) > 1:
            if _keymatch(a[1:], "outfile", 4):
                if i + 1 >= len(args):
                    print("djpeg: missing argument for -outfile", file=sys.stderr)
                    return 1
                outfile = args[i + 1]; i += 2; continue
            switches.append(a)
            if (_keymatch(a[1:], "scale", 1) or _keymatch(a[1:], "dct", 2)) and i + 1 < len(args):
                switches.append(args[i + 1]); i += 1
        else:
            files.append(a)
        i += 1
    try:
        opts = parse(switches)
    except (NotOnDevice, ValueError) as e:
        print(f"djpeg: {e}", file=sys.stderr)
        return 1
    if len(files) != 1:
        print("usage: python -m mozjpeg_b200.djpeg [switches] [-outfile name] file.jpg", file=sys.stderr)
        return 2
    with open(files[0], "rb") as f:
        src = f.read()
    enc = Encoder(0)
    try:
        px = enc.decompress([src], **opts)[0]
    finally:
        enc.close()
    out = ppm_bytes(px)
    if outfile:
        with open(outfile, "wb") as fo:
            fo.write(out)
    else:
        sys.stdout.buffer.write(out)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
