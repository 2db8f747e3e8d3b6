"""Synthetic benchmark/test inputs (SURVEY 8d).  Pure numpy; no encoder logic."""
import numpy as np


def synth_image(seed: int, width: int, height: int) -> np.ndarray:
    """SURVEY 8(d) synthetic input: smooth sinusoid field per channel (periods
    33-143 px) + N(0, 12) noise, clipped, plus a saturated white rectangle with
    thin black lines (~1% of the area) to exercise deringing."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:height, 0:width].astype(np.float32)
    img = np.empty((height, width, 3), dtype=np.float32)
    for c in range(3):
        px, py = rng.uniform(33, 143, 2)
        ph = rng.uniform(0, 6.28, 2)
        amp = rng.uniform(40, 90)
        img[..., c] = 128 + amp * np.sin(x * (6.2831853 / px) + ph[0]) * np.cos(y * (6.2831853 / py) + ph[1])
    img += rng.normal(0, 12, img.shape).astype(np.float32)
    out = np.clip(img, 0, 255).astype(np.uint8)
    rw, rh = max(8, width // 10), max(8, height // 10)
    x0 = int(rng.integers(0, max(1, width - rw))); y0 = int(rng.integers(0, max(1, height - rh)))
    out[y0:y0 + rh, x0:x0 + rw] = 255
    out[y0 + rh // 3:y0 + rh // 3 + 1, x0:x0 + rw] = 0
    out[y0:y0 + rh, x0 + rw // 2:x0 + rw // 2 + 1] = 0
    return out


def synth_image12(seed: int, width: int, height: int) -> np.ndarray:
    """12-bit variant (SURVEY 8d, config 5): the 8-bit generator x16 plus uniform{0..15},
    uint16 samples in [0, 4095]."""
    base = synth_image(seed, width, height).astype(np.uint16) * 16
    rng = np.random.default_rng(seed + 7919)
    return (base + rng.integers(0, 16, base.shape, dtype=np.uint16)).astype(np.uint16)


def synth_planes(p, seed: int):
    """Raw-data test input (jpeg_write_raw_data): one (hib*8, wib*8) uint8 plane per component of the
    parameter block p, smooth field + noise, already 'downsampled'."""
    rng = np.random.default_rng(seed)
    nc = p.num_components
    hmax = max(p.comp_info[i].h_samp_factor for i in range(nc)); vmax = max(p.comp_info[i].v_samp_factor for i in range(nc))
    out = []
    for ci in range(nc):
        h = p.comp_info[ci].h_samp_factor; v = p.comp_info[ci].v_samp_factor
        wib = -(-p.image_width * h // (hmax * 8)); hib = -(-p.image_height * v // (vmax * 8))
        yy, xx = np.mgrid[0:hib * 8, 0:wib * 8]
        a = 128 + 90 * np.sin(xx / (7 + 3 * ci)) * np.cos(yy / (9 + 2 * ci)) + rng.normal(0, 10, (hib * 8, wib * 8))
        out.append(np.clip(a, 0, 255).astype(np.uint8))
    return out


def synth_image16(seed: int, width: int, height: int, channels: int = 1) -> np.ndarray:
    """16-bit input for the lossless encoder (medical / scientific content): a smooth field over the full 0..65535
    range per channel plus N(0, 64) noise, clipped; uint16 samples, (height, width, channels)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:height, 0:width].astype(np.float32)
    out = np.empty((height, width, channels), dtype=np.uint16)
    for c in range(channels):
        px, py = rng.uniform(200, 900, 2)
        ph = rng.uniform(0, 6.28, 2)
        f = 32768 + 30000 * np.sin(x * (6.2831853 / px) + ph[0]) * np.cos(y * (6.2831853 / py) + ph[1])
        out[..., c] = np.clip(f + rng.normal(0, 64, f.shape).astype(np.float32), 0, 65535).astype(np.uint16)
    return out
