"""tjbench -lossless on one 3840x2160 image, with the libjpeg interposer preloaded (device path) and without it (the
reference's C encoder), alternating in one session.  One JSON line per workload with the Mpixels/s tjbench prints for
every run, whether the two runs wrote the same file, and the card's name, power limit and clocks read in the same run.

    python tools/bench_tjbench_lossless.py [--rounds 3] [--benchtime 5]

tjbench takes its pixel format from the command line (BGR by default) and converts grey input to it, so its 16-bit
workload here is 16-bit RGB.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TJBENCH = os.path.join(ROOT, "oracle", "_ref", "tjbench")
SHIM = os.path.join(ROOT, "integration", "_build", "libjpeg_b200shim.so")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else None


def write_ppm(path, prec, w=3840, h=2160, seed=7):
    """Smooth gradients plus a few bits of noise per sample, seeded."""
    rng = np.random.default_rng(seed)
    top = (1 << prec) - 1
    yy, xx = np.mgrid[0:h, 0:w]
    base = ((xx * 3 + yy * 2) * (top // 4096 + 1))[..., None] + np.arange(3) * 31
    a = (base + rng.integers(0, 64, size=(h, w, 3))) % (top + 1)
    data = a.astype(">u2").tobytes() if prec > 8 else a.astype(np.uint8).tobytes()
    with open(path, "wb") as f:
        f.write(b"P6\n%d %d\n%d\n" % (w, h, top) + data)


def tjbench(d, psv, prec, benchtime, device):
    env = dict(os.environ, LD_PRELOAD=SHIM, B200_SHIM_REQUIRE="1") if device else dict(os.environ)
    r = subprocess.run([TJBENCH, "img.ppm", str(psv), "-precision", str(prec), "-lossless", "-componly", "-benchtime", str(benchtime),
                        "-warmup", "1"], cwd=d, env=env, capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        sys.exit(f"tjbench failed ({'device' if device else 'reference'}): {r.stdout[-2000:]}{r.stderr[-2000:]}")
    mp = float(re.search(r"Throughput:\s+([0-9.]+) Megapixels/sec", r.stdout).group(1))
    jpg = [f for f in os.listdir(d) if f.endswith(".jpg")][0]
    with open(os.path.join(d, jpg), "rb") as f:
        data = f.read()
    os.remove(os.path.join(d, jpg))
    return mp, data


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--benchtime", type=float, default=5)
    a = ap.parse_args()
    gpu = card()
    for name, prec, psv in (("16-bit RGB 3840x2160, PSV 1", 16, 1), ("8-bit RGB 3840x2160, PSV 1", 8, 1)):
        with tempfile.TemporaryDirectory() as d:
            write_ppm(os.path.join(d, "img.ppm"), prec)
            dev, ref, same = [], [], True
            for _ in range(a.rounds):
                mp_d, out_d = tjbench(d, psv, prec, a.benchtime, True)
                mp_r, out_r = tjbench(d, psv, prec, a.benchtime, False)
                dev.append(mp_d); ref.append(mp_r); same = same and out_d == out_r
            print(json.dumps({"workload": name, "device_mpix_s": dev, "reference_mpix_s": ref, "same_file": same,
                              "speedup_median": float(np.median(dev) / np.median(ref)), "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
