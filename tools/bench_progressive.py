"""Decoding progressive JPEG files on the device, on N seeded 3840x2160 4:2:0 sources written by the device encoder with
mozjpeg's default profile (progressive, scan search) at -quality 75 and 90.  Two more sets carry -restart 1; the
default profile's scan search writes such files with one restart interval for all scans (the reference decoder warns
on them and the device refuses them), so those sets use the standard progressive script (-revert -progressive), whose
scans carry their own DRI.  Prints JSON lines, each with the card's name, power limit and SM clock read in this run:
  decode     : Encoder.read_coefficients: the stage times per image, refinements separate (dec_dc_refine,
               dec_ac_refine), and last_decode_sync
  jpegtran   : default and -rotate 90, file bytes to file bytes (Encoder with progressive decode on)
  djpeg      : default and -scale 1/4, pixels left in HBM
  cjpeg      : -quality 75 from the JPEG files
  ref        : the reference's jpegtran on the host threads, where oracle/_ref is present
The first and last output of each route are compared with the reference's (jpegtran binary, build/librefdec.so pixels)
where it is present.  There is no CPU fallback: without a CUDA device the script fails.

    python tools/bench_progressive.py [--n 64] [--reps 3]
"""
import argparse
import hashlib
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

SETS = (("default_q75", ["-quality", "75"]), ("default_q90", ["-quality", "90"]),
        ("standard_q75_restart_1", ["-revert", "-progressive", "-quality", "75", "-restart", "1"]),
        ("standard_q90_restart_1", ["-revert", "-progressive", "-quality", "90", "-restart", "1"]))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"card": r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"}


def timed(fn, reps):
    """the output of a warm-up call, then the spread of reps timed calls"""
    out = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    ts.sort()
    return ts, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--sets", default=",".join(s for s, _ in SETS))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_progressive.py needs a CUDA device")
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    import recompress_cases as R
    from oracle import oracle as O
    W, H, N = 3840, 2160, a.n
    enc = mj.Encoder(0)
    enc.set_progressive_decode(True)
    pool = ThreadPoolExecutor(a.threads)
    ref_tran = os.path.join(O.REF_DIR, "jpegtran")
    have_ref = os.path.exists(ref_tran) and R.have_reference()
    imgs = list(pool.map(lambda i: O.synth_image(2000 + i, W, H), range(N)))          # the same pictures in every set
    for sset, sw in SETS:
        if sset not in a.sets.split(","):
            continue
        p = mj.params_from_switches(sw, W, H, 3)
        srcs = []
        for i0 in range(0, N, 8):
            srcs += enc.encode_batch(p, np.stack(imgs[i0:i0 + 8]))
        base = dict(card(), set=sset, switches=sw, images=N, width=W, height=H, source_mb=round(sum(map(len, srcs)) / 1e6, 1))
        # decode stage times
        st = []
        for _ in range(1 + a.reps):
            enc.read_coefficients(srcs)
            st.append(enc.stage_times())
        st = st[1:]
        stages = {k: round(sorted(s[k] for s in st)[len(st) // 2] / N, 4) for k in st[0]}
        totals = sorted(sum(s.values()) / N for s in st)
        rounds, redone = enc.last_decode_sync()
        print(json.dumps(dict(base, what="decode", stage_ms_per_image=stages, total_ms_per_image=round(sum(stages.values()), 4),
                              total_ms_per_image_min_max=[round(totals[0], 4), round(totals[-1], 4)], reps=len(st), max_cta_rounds=rounds, resync_subsequences=redone)), flush=True)
        outs = {}
        for name, fn in (("jpegtran", lambda: T.transcode(enc, srcs, None, [])),
                         ("jpegtran -rotate 90", lambda: T.transcode(enc, srcs, None, ["-rotate", "90"])),
                         ("djpeg", lambda: enc.decompress(srcs)),
                         ("djpeg -scale 1/4", lambda: enc.decompress(srcs, scale=(1, 4))),
                         ("cjpeg -quality 75", lambda: enc.recompress(mj.params_for_jpeg_input(["-quality", "75"], srcs[0]), srcs))):
            ts, outs[name] = timed(fn, a.reps)
            t = ts[len(ts) // 2]
            print(json.dumps(dict(base, what="route", route=name, images_per_s=round(N / t, 2), ms_median=round(t * 1e3, 1),
                                  ms_min=round(ts[0] * 1e3, 1), ms_max=round(ts[-1] * 1e3, 1), reps=len(ts))), flush=True)
        if have_ref:
            for tsw in ([], ["-rotate", "90"]):
                t0 = time.perf_counter()
                want = list(pool.map(lambda s: subprocess.run([ref_tran, *tsw], input=s, capture_output=True, check=True).stdout, srcs))
                t = time.perf_counter() - t0
                print(json.dumps(dict(base, what="ref", route="jpegtran " + " ".join(tsw), host_threads=a.threads, images_per_s=round(N / t, 2))), flush=True)
                got = outs["jpegtran" + (" -rotate 90" if tsw else "")]
                assert all(got[i] == want[i] for i in (0, N - 1)), f"jpegtran {tsw}: device output differs from the reference's"
            for i in (0, N - 1):
                assert hashlib.md5(outs["djpeg"][i].tobytes()).digest() == hashlib.md5(R.ref_decompress(srcs[i])[0].tobytes()).digest(), "pixels differ"
            print(json.dumps(dict(base, what="check", first_and_last_outputs_identical_to="reference jpegtran and decompressor")), flush=True)
    enc.close()
    pool.shutdown()


if __name__ == "__main__":
    main()
