"""jpegtran from file bytes on the device against today's routes, on N seeded 3840x2160 4:2:0 sources written with the
reference's settings -revert -quality 90 (by the CPU oracle, bit-identical to the reference's cjpeg), once without
restarts and once with -restart 1.  Routes, per workload (jpegtran default, -progressive, -optimize):
  device : Encoder.transcode_files (device entropy decode + re-encode) from host file bytes
  host   : the reference's jpeg_read_coefficients on the host threads, then Encoder.encode_batch_coefs
  ref    : the reference's own jpegtran binary on the host threads
Every output is checked byte for byte against the reference's jpegtran.  Prints the card, its power limit and SM clock,
the decode stage times per image and the synchronisation work, then one line per (source set, workload, route).

    python tools/bench_transcode.py [--n 64] [--reps 3] [--sets no_restart,restart_1]
"""
import argparse
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--sets", default="no_restart,restart_1")
    a = ap.parse_args()
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    W, H = 3840, 2160
    print("card:", card(), "| host threads:", a.threads, flush=True)
    enc = mj.Encoder(0)
    pool = ThreadPoolExecutor(a.threads)
    for sset, sw in (("no_restart", ["-revert", "-quality", "90"]), ("restart_1", ["-revert", "-quality", "90", "-restart", "1"])):
        if sset not in a.sets.split(","):
            continue
        p = mj.params_from_switches(sw, W, H, 3)
        srcs = [O.oracle_encode(p, O.synth_image(1000 + i, W, H)).jpeg for i in range(a.n)]
        mb = sum(len(s) for s in srcs) / 1e6
        planes = enc.read_coefficients(srcs)                           # warm-up + decode stage times
        st = enc.stage_times()
        rounds, redone = enc.last_decode_sync()
        dec = {k: v / a.n for k, v in st.items() if k.startswith("dec_")}
        print(f"[{sset}] {a.n} sources, {mb:.1f} MB; decode ms/image: " + " ".join(f"{k}={v:.4f}" for k, v in dec.items())
              + f" total={sum(dec.values()):.4f}; max CTA rounds={rounds}, cross-CTA re-decoded subsequences={redone}", flush=True)
        for tsw in ([], ["-progressive"], ["-optimize"]):
            t0 = time.perf_counter()
            want = list(pool.map(lambda s: O.ref_jpegtran(s, tsw), srcs))
            t = time.perf_counter() - t0
            print(f"[{sset}] jpegtran {' '.join(tsw) or 'default':13s} ref   : {a.n / t:8.1f} images/s {a.n * W * H / t / 1e6:9.1f} MP/s"
                  f"  ({t * 1e3:.1f} ms per batch, one run)", flush=True)
            pt, prefer = T.params_for_transcode(T.parse_header(srcs[0]), tsw)

            def device():
                return T.transcode(enc, srcs, None, tsw)

            def host():
                coefs = list(pool.map(lambda s: O.ref_read_coefs(s)["coefs"], srcs))
                stacked = [np.stack([c[ci] for c in coefs]) for ci in range(len(coefs[0]))]
                return T.transcode(enc, srcs, stacked, tsw)

            for name, fn in (("device", device), ("host", host)):
                out = fn()
                assert out == want, (sset, tsw, name, "output differs from the reference's jpegtran")
                ts = []
                for _ in range(a.reps):
                    t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
                t = min(ts)
                print(f"[{sset}] jpegtran {' '.join(tsw) or 'default':13s} {name:6s}: {a.n / t:8.1f} images/s {a.n * W * H / t / 1e6:9.1f} MP/s"
                      f"  ({t * 1e3:.1f} ms per batch, best of {a.reps}; byte-identical)", flush=True)
    enc.close()
    pool.shutdown()


if __name__ == "__main__":
    main()
