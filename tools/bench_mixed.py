"""Batches of mixed geometry (Encoder.decompress_mixed / recompress_mixed) against a loop of one-file calls and against one
call per geometry group, on a seeded corpus of common photo sizes: 640x480, 1280x720, 1920x1080, 2048x1536, 3024x4032
portrait, 4000x3000, 3840x2160 and the ragged 1001x667 and 333x500, in 4:2:0, 4:4:4 and gray, qualities 75 .. 95, with
and without -restart 1, and a progressive subset with -restart 1 (decoded with progressive decode on).  The sources are written by the
device encoder from the CPU oracle's seeded pixels; nothing is read from disk.  Host file bytes in, host pixels or file
bytes out throughout.  Prints JSON lines, each carrying the card's name, power limit and SM clock read in this run:
  corpus   : images, megapixels, distinct geometries
  decompress / ladder : per route (mixed, single, groups) images/s, megapixels/s, median and spread of the call time,
             and for the mixed route its stage times and kernel launches per call.  The ladder is 1/1 -quality 80 and
             1/4 -quality 75 (recompress_mixed against recompress_renditions per file and per geometry group).
  check    : every mixed output byte-identical to the single calls' (the script asserts it)
There is no CPU fallback: without a CUDA device the encoder cannot be created and the script fails.

    python tools/bench_mixed.py [--n 96] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(640, 480), (1280, 720), (1920, 1080), (2048, 1536), (3024, 4032), (4000, 3000), (3840, 2160), (1001, 667), (333, 500)]
LAYOUTS = [["-sample", "2x2"], ["-sample", "1x1"], ["-grayscale"]]
LADDER = [(["-quality", "80"], {}), (["-quality", "75"], dict(scale=(1, 4)))]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    f = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")] if r.stdout.strip() else []
    return {"card": f[0], "power_limit": f[1], "sm_clock": f[2]} if len(f) == 3 else {"card": "unknown"}


def corpus(enc, n, seed=2026):
    """n sources: size, layout, quality, restarts and progressive drawn from a seeded generator"""
    import mozjpeg_b200 as mj
    from mozjpeg_b200 import jpegtran as T
    from oracle import oracle as O
    rng = np.random.default_rng(seed)
    files, keys, px_cache = [], [], {}
    for i in range(n):
        w, h = SIZES[i % len(SIZES)]
        lay = LAYOUTS[int(rng.integers(len(LAYOUTS)))]
        q = int(rng.integers(75, 96))
        # the progressive subset is the standard script with restarts: without them the serial AC refinement walk
        # (about 1 s per 4K image) would be all the benchmark measures
        prog = rng.random() < 0.2
        rst = prog or rng.random() < 0.3
        sw = ["-revert"] + (["-progressive"] if prog else []) + ["-quality", str(q)] + lay + (["-restart", "1"] if rst else [])
        if (w, h) not in px_cache:
            px_cache[(w, h)] = O.synth_image(seed + len(px_cache), w, h)
        files.append(enc.encode_batch(mj.params_from_switches(sw, w, h, 3), px_cache[(w, h)][None])[0])
        # the geometry the one-geometry calls compare (a gray file may carry 2x1 sampling factors, as cjpeg writes them)
        s = T.parse_source(files[-1])
        keys.append((w, h, s.num_components, s.jpeg_color_space, tuple((s.h_samp_factor[c], s.v_samp_factor[c]) for c in range(s.num_components))))
    return files, keys


def timed(fn, reps):
    fn()                                                           # warm-up: every shape of the timed calls
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); out = fn(); ts.append(time.perf_counter() - t0)
    return out, ts


def line(base, what, route, ts, n, mp, **kw):
    t = sorted(ts)[len(ts) // 2]
    return json.dumps(dict(base, what=what, route=route, images_per_s=round(n / t, 2), mpixels_per_s=round(mp / t, 1), ms_median=round(t * 1e3, 1),
                           ms_min=round(min(ts) * 1e3, 1), ms_max=round(max(ts) * 1e3, 1), reps=len(ts), **kw))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=96)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_mixed.py needs a CUDA device")
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    enc.set_progressive_decode(True)
    files, keys = corpus(enc, a.n)
    n = len(files)
    mp = sum(k[0] * k[1] for k in keys) / 1e6
    groups = {}
    for i, k in enumerate(keys):
        groups.setdefault(k, []).append(i)
    base = dict(card(), images=n, megapixels=round(mp, 1))
    print(json.dumps(dict(base, what="corpus", geometries=len(groups), source_mb=round(sum(map(len, files)) / 1e6, 1))), flush=True)

    # decompress, one default rung
    def mixed_dec():
        return enc.decompress_mixed(files)[0]

    def single_dec():
        return [enc.decompress([f])[0] for f in files]

    def group_dec():
        out = [None] * n
        for idx in groups.values():
            got = enc.decompress([files[i] for i in idx])
            for j, i in enumerate(idx):
                out[i] = got[j]
        return out

    outs = {}
    for name, fn in (("mixed", mixed_dec), ("single", single_dec), ("groups", group_dec)):
        before = enc.kernel_launches()
        outs[name], ts = timed(fn, a.reps)
        launches = (enc.kernel_launches() - before) / (a.reps + 1)
        extra = dict(kernel_launches_per_call=launches)
        if name == "mixed":
            extra["stage_ms"] = {k: round(v, 3) for k, v in enc.stage_times().items()}
        print(line(base, "decompress", name, ts, n, mp, **extra), flush=True)
    same_dec = all(np.array_equal(outs["mixed"][i], outs[r][i]) for r in ("single", "groups") for i in range(n))

    # a 1/1 q80 + 1/4 q75 rendition ladder
    def mixed_lad():
        return enc.recompress_mixed(files, LADDER)

    def single_lad():
        return [enc.recompress_renditions([f], [(mj.params_for_jpeg_input(sw, f, **kw), kw) for sw, kw in LADDER]) for f in files]

    def group_lad():
        out = [[None] * n for _ in LADDER]
        for idx in groups.values():
            gf = [files[i] for i in idx]
            got = enc.recompress_renditions(gf, [(mj.params_for_jpeg_input(sw, gf[0], **kw), kw) for sw, kw in LADDER])
            for r in range(len(LADDER)):
                for j, i in enumerate(idx):
                    out[r][i] = got[r][j]
        return out

    lad = {}
    for name, fn in (("mixed", mixed_lad), ("single", single_lad), ("groups", group_lad)):
        before = enc.kernel_launches()
        lad[name], ts = timed(fn, a.reps)
        launches = (enc.kernel_launches() - before) / (a.reps + 1)
        extra = dict(kernel_launches_per_call=launches)
        if name == "mixed":
            extra["stage_ms"] = {k: round(v, 3) for k, v in enc.stage_times().items()}
        print(line(base, "ladder", name, ts, n, mp, **extra), flush=True)
    single_files = [[lad["single"][i][r][0] for i in range(n)] for r in range(len(LADDER))]
    same_lad = lad["mixed"] == single_files and lad["mixed"] == lad["groups"]
    print(json.dumps(dict(base, what="check", decompress_byte_identical_to_single_and_group_calls=same_dec,
                          ladder_byte_identical_to_single_and_group_calls=same_lad)), flush=True)
    enc.close()
    assert same_dec and same_lad, "a mixed output differs from the single calls'"


if __name__ == "__main__":
    main()
