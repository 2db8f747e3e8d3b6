#!/usr/bin/env python3
"""Per-image quantization tables on device-resident 3840x2160 RGB input, -baseline -sample 2x2 with the trellis on:

  1. ladder: one image at 8 qualities (40, 50, ..., 90, 95) as one b200jpeg_encode_batch_qtables call with image stride
     0, against 8 encode_batch calls, one per quality (ms best / median after warm-up, host clock around synchronised
     calls, the files read back as a user would);
  2. mixed batch: N images whose tables cycle through those 8 qualities, against the same batch through encode_batch
     at quality 75 (GP/s, CUDA events);
  3. parity: every ladder file and the first and last file of (2) against the reference (oracle/_ref), where built.

Prints one JSON line with the GPU name, SM count and power limit read in the same run.

    python tools/bench_qladder.py [--images 256] [--iters 5] [--warmup 2]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mozjpeg_b200 as mj  # noqa: E402
from oracle import oracle as O  # noqa: E402
from bench_colorspaces import power_limit_w  # noqa: E402

QUALITIES = (40, 50, 60, 70, 80, 85, 90, 95)
BASE = ["-baseline", "-sample", "2x2"]


def timed(fn, iters, warmup, events=False):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        if events:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        else:
            t0 = time.perf_counter(); fn(); torch.cuda.synchronize()
            ms.append((time.perf_counter() - t0) * 1e3)
    return min(ms), float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    w, h, n = a.width, a.height, a.images
    enc = mj.Encoder(0)
    p = mj.params_from_switches(BASE, w, h, 3)
    ladder = mj.quality_tables(p, QUALITIES)
    res = {"bench": "qladder", "width": w, "height": h, "switches": " ".join(BASE), "qualities": list(QUALITIES)}
    have_ref = O.ref_available()

    # 1. ladder
    img = O.synth_image(1000, w, h)
    dev = torch.from_numpy(img).cuda()
    st = dev.stride()
    singles = []
    for q in ladder:
        pq = p.copy(); np.ctypeslib.as_array(pq.quant_tbl)[:] = q
        singles.append(pq)

    def one_call():
        enc.encode_batch_qtables_ptr(p, dev.data_ptr(), True, st[0], 0, ladder)
        return [enc.get_output(i) for i in range(len(ladder))]

    def eight_calls():
        out = []
        for pq in singles:
            enc.encode_batch_ptr(pq, dev.data_ptr(), True, st[0], st[0] * h, 1)
            out.append(enc.get_output(0))
        return out

    b1, m1 = timed(one_call, a.iters, a.warmup)
    b8, m8 = timed(eight_calls, a.iters, a.warmup)
    files = one_call()
    res["ladder"] = {"one_call_ms_best": round(b1, 2), "one_call_ms_median": round(m1, 2),
                     "eight_calls_ms_best": round(b8, 2), "eight_calls_ms_median": round(m8, 2),
                     "same_files_as_eight_calls": files == eight_calls(),
                     "match_reference": ([O.ref_encode(img, ["-baseline", "-quality", str(q), "-sample", "2x2"]) for q in QUALITIES] == files) if have_ref else None}
    del dev

    # 2. mixed batch
    distinct = [O.synth_image(1000 + i, w, h) for i in range(8)]
    bat = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
    for i in range(n):
        bat[i] = torch.from_numpy(distinct[i % 8])
    torch.cuda.synchronize()
    bs = bat.stride()
    qt = ladder[np.arange(n) % len(QUALITIES)]
    p75 = mj.params_from_switches(["-baseline", "-quality", "75", "-sample", "2x2"], w, h, 3)
    bm, mm = timed(lambda: enc.encode_batch_qtables_ptr(p, bat.data_ptr(), True, bs[1], bs[0], qt), a.iters, a.warmup, events=True)
    first_last = [enc.get_output(0), enc.get_output(n - 1)]
    bq, mq = timed(lambda: enc.encode_batch_ptr(p75, bat.data_ptr(), True, bs[1], bs[0], n), a.iters, a.warmup, events=True)
    gp = lambda ms: round(n * w * h / (ms * 1e-3) / 1e9, 2)
    ok = None
    if have_ref:
        ok = first_last == [O.ref_encode(distinct[i % 8], ["-baseline", "-quality", str(QUALITIES[i % len(QUALITIES)]), "-sample", "2x2"]) for i in (0, n - 1)]
    res["mixed"] = {"images": n, "per_image_gpix_per_s": gp(bm), "per_image_ms_best": round(bm, 2), "per_image_ms_median": round(mm, 2),
                    "q75_gpix_per_s": gp(bq), "q75_ms_best": round(bq, 2), "q75_ms_median": round(mq, 2), "first_last_match_reference": ok}
    prop = torch.cuda.get_device_properties(0)
    res.update(gpu=prop.name, sms=prop.multi_processor_count, power_limit_w=power_limit_w())
    print(json.dumps(res))
    enc.close()


if __name__ == "__main__":
    main()
