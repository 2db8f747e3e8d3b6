"""jpegtran's lossless transforms on the device, from file bytes, on N seeded 3840x2160 4:2:0 sequential sources written
with the reference's settings -revert -quality 90 (by the CPU oracle, like tools/bench_transcode.py).  Workloads: no
transform, -rotate 90, -rotate 90 -trim, -crop 1920x1080+960+540 and -grayscale, each under jpegtran's default
profile (scan search) and with -optimize; and the reference's own jpegtran -rotate 90 on the host threads.  Every
device output is checked byte for byte against the reference's jpegtran where its build is present.  Prints the card,
its power limit and SM clock (read in the same run), then per workload img/s end to end and the `forward` stage (on
the coefficient route: the coefficient import, where the transform is applied) per image.

    python tools/bench_transform.py [--n 64] [--reps 3] [--threads 16]
"""
import argparse
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [[], ["-rotate", "90"], ["-rotate", "90", "-trim"], ["-crop", "1920x1080+960+540"], ["-grayscale"]]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--identity-only", action="store_true", help="only the untransformed route (runs on trees without transforms)")
    a = ap.parse_args()
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    W, H = 3840, 2160
    have_ref = os.path.exists(os.path.join(O.REF_DIR, "jpegtran"))
    pool = ThreadPoolExecutor(a.threads)
    p = mj.params_from_switches(["-revert", "-quality", "90"], W, H, 3)
    srcs = list(pool.map(lambda i: O.oracle_encode(p, O.synth_image(1000 + i, W, H)).jpeg, range(a.n)))
    enc = mj.Encoder(0)
    print("card (name, power limit, SM clock, max SM clock):", card(), "| host threads:", a.threads, flush=True)
    for prof in ([], ["-optimize"]):
        for xf in WORKLOADS[:1] if a.identity_only else WORKLOADS:
            sw = xf + prof
            out = T.transcode(enc, srcs, None, sw)                  # warm-up
            if have_ref:
                want = list(pool.map(lambda s: O.ref_jpegtran(s, sw), srcs))
                assert out == want, (sw, "output differs from the reference's jpegtran")
            ts, fwd = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter(); T.transcode(enc, srcs, None, sw); ts.append(time.perf_counter() - t0)
                fwd.append(enc.stage_times().get("forward", float("nan")))
            t = min(ts)
            print(f"jpegtran {' '.join(sw) or 'default':38s} device: {a.n / t:7.1f} img/s ({t * 1e3:8.1f} ms per batch, best of {a.reps})"
                  f"  forward {min(fwd) / a.n * 1e3:7.1f} us/image{'  byte-identical' if have_ref else ''}", flush=True)
    if have_ref and not a.identity_only:
        t0 = time.perf_counter()
        list(pool.map(lambda s: O.ref_jpegtran(s, ["-rotate", "90"]), srcs))
        t = time.perf_counter() - t0
        print(f"jpegtran {'-rotate 90':38s} ref   : {a.n / t:7.1f} img/s ({t * 1e3:8.1f} ms per batch, one run, {a.threads} threads)", flush=True)
    print("card after:", card(), flush=True)
    enc.close()
    pool.shutdown()


if __name__ == "__main__":
    main()
