"""Lossless (SOF3) throughput of device-resident batches, one JSON line per workload:
  * 64 x 3840x2160 16-bit grayscale, predictors 1 and 6;
  * 64 x 3840x2160 8-bit RGB, predictor 1.
Each line holds GP/s and ms per batch (best and median over --steps timed batches, device pipeline only), the per-stage
times of b200jpeg_last_stage_times, whether the first and last files equal the reference's bytes, the reference's C
encoder on the host threads for the same images, and the card's name, SM count and power limit read in the same run.

    python tools/bench_lossless.py [--steps 5] [--warmup 1] [--images 64]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import torch
    prop = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"name": prop.name, "sms": prop.multi_processor_count, "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def images(n, h, w, nc, prec, seed=7):
    """Smooth gradients plus noise (a few bits per sample), seeded."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    top = (1 << prec) - 1
    base = ((xx * 3 + yy * 2) * (top // 4096 + 1)) % (top + 1)
    out = np.empty((n, h, w, nc), dtype=np.uint8 if prec == 8 else np.uint16)
    for i in range(n):
        for c in range(nc):
            out[i, :, :, c] = (base + i * 97 + c * 31 + rng.integers(0, 64, size=(h, w))) % (top + 1)
    return out


def run(enc, name, sw, imgs, steps, warmup):
    import torch
    import mozjpeg_b200 as mj
    import test_lossless as T
    n, h, w, nc = imgs.shape
    p = mj.params_from_switches(sw, w, h, nc)
    t = torch.from_numpy(imgs.view(np.int16) if imgs.dtype == np.uint16 else imgs).cuda()
    pitch, stride = imgs.strides[1], imgs.strides[0]
    for _ in range(warmup):
        enc.encode_batch_ptr(p, t.data_ptr(), True, pitch, stride, n, device_only=True)
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        t0 = time.perf_counter()
        enc.encode_batch_ptr(p, t.data_ptr(), True, pitch, stride, n, device_only=True)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    stages = enc.stage_times()
    enc.encode_batch_ptr(p, t.data_ptr(), True, pitch, stride, n)              # with the files, for the parity check
    files = [enc.get_output(0), enc.get_output(n - 1)]
    in_cs = mj._abi.CS_GRAYSCALE if nc == 1 else mj._abi.CS_RGB
    ref = [T.ref_encode(imgs[0], sw, in_cs), T.ref_encode(imgs[n - 1], sw, in_cs)]
    threads = os.cpu_count() or 1
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda i: T.ref_encode(imgs[i], sw, in_cs), range(n)))
    ref_s = time.perf_counter() - t0
    gp = n * w * h / 1e9
    best, med = min(ms), float(np.median(ms))
    return {"workload": name, "switches": " ".join(sw), "images": n, "width": w, "height": h,
            "gpps_best": gp / (best / 1e3), "gpps_median": gp / (med / 1e3), "ms_best": best, "ms_median": med,
            "stage_ms": stages, "parity_first_last": files == ref, "jpeg_bytes_first": len(files[0]),
            "reference_host_threads": threads, "reference_host_s": ref_s, "reference_host_gpps": gp / ref_s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--images", type=int, default=64)
    a = ap.parse_args()
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    info = card()
    from mozjpeg_b200.synth import synth_image16
    gray16 = np.stack([synth_image16(1000 + i, 3840, 2160) for i in range(a.images)])
    for psv in (1, 6):
        r = run(enc, f"gray16_psv{psv}", ["-revert", "-precision", "16", "-lossless", str(psv)], gray16, a.steps, a.warmup)
        r["card"] = info
        print(json.dumps(r), flush=True)
    del gray16
    rgb8 = images(a.images, 2160, 3840, 3, 8)
    r = run(enc, "rgb8_psv1", ["-revert", "-lossless", "1"], rgb8, a.steps, a.warmup)
    r["card"] = info
    print(json.dumps(r), flush=True)
    enc.close()


if __name__ == "__main__":
    main()
