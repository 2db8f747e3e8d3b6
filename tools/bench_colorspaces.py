#!/usr/bin/env python3
"""Device-resident throughput of the 4-component encodes next to RGB->YCbCr, at the TurboJPEG defaults (quality 75,
4:2:0, JCP_FASTEST): a batch of N x 3840x2160 images timed with CUDA events after warm-up, for CMYK->YCCK, CMYK->CMYK
and RGB->YCbCr.  The first and last image of every batch are byte-checked against the reference's tj3Compress8
(build/librefcs.so over oracle/_ref).  Prints one JSON line: GP/s per conversion, GPU name, SM count, power limit.

    python tools/bench_colorspaces.py [--images 64] [--iters 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mozjpeg_b200 as mj  # noqa: E402
import colorspace_cases as CC  # noqa: E402


def power_limit_w():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:
        import subprocess
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
            return float(out.splitlines()[0])
        except Exception:
            return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    w, h, n = a.width, a.height, a.images
    enc = mj.Encoder(0)
    res = {"bench": "colorspaces", "images": n, "width": w, "height": h, "settings": "TurboJPEG defaults: quality 75, 4:2:0, JCP_FASTEST"}
    for name, ic, params in (("cmyk_ycck", 4, mj.tj3_params(w, h, 75, "420", cmyk=True)),
                             ("cmyk_cmyk", 4, mj.tj3_params(w, h, 75, "420", cmyk=True, colorspace=mj._abi.CS_CMYK)),
                             ("rgb_ycbcr", 3, mj.tj3_params(w, h, 75, "420"))):
        base = np.stack([CC.cmyk_image(1, w, h, ic), CC.cmyk_image(2, w, h, ic)])
        dev = torch.empty((n, h, w, ic), dtype=torch.uint8, device="cuda")
        dev[:] = torch.from_numpy(base[0])
        dev[-1] = torch.from_numpy(base[1])
        torch.cuda.synchronize()
        st = dev.stride()
        run = lambda: enc.encode_batch_ptr(params, dev.data_ptr(), True, st[1], st[0], n)
        for _ in range(a.warmup):
            run()
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        ok = None                                     # RGB->YCbCr at these settings is pinned by the existing suite
        cs = {"cmyk_ycck": -1, "cmyk_cmyk": 3}.get(name)
        if cs is not None and CC.have_reference():
            refs = [CC.ref_encode_tj(img, 75, 2, 0, 0, cs) for img in base]
            ok = refs == [enc.get_output(0), enc.get_output(n - 1)]
        best = min(ms)
        res[name] = {"ms_best": round(best, 2), "ms_median": round(float(np.median(ms)), 2),
                     "gpix_per_s": round(n * w * h / (best * 1e-3) / 1e9, 2), "first_last_match_reference": ok}
        del dev
        torch.cuda.empty_cache()
    prop = torch.cuda.get_device_properties(0)
    res.update(gpu=prop.name, sms=prop.multi_processor_count, power_limit_w=power_limit_w())
    print(json.dumps(res))
    enc.close()


if __name__ == "__main__":
    main()
