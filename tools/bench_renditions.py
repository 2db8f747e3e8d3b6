"""A rendition ladder from one device decode (Encoder.recompress_renditions) against one recompress call per rung, on N
seeded 3840x2160 4:2:0 sources written by the CPU oracle, in three sets: sequential without restarts, sequential with
-restart 1, and mozjpeg's default progressive profile (decoded with progressive decode on).  The ladder:
    1/1 -quality 80 -sample 2x2,  1/2 -quality 80 -sample 2x2,  1/4 -quality 75 -sample 2x2,  1/8 -quality 70 -sample 2x2
Host file bytes to host file bytes throughout.  Prints JSON lines, each carrying the card's name, power limit and SM
clock read in this run:
  ladder    : Encoder.recompress_renditions, source images per second, and its stage times per image
  separate  : four Encoder.recompress calls, one per rung, source images per second
  ref       : where oracle/_ref is available, the reference library's scaled decode (tests/refdecopt.c) and then the
              reference's cjpeg on the PPM, per rung, on the host threads
  check     : every ladder file byte-identical to the separate calls' and, where the reference exists, to the
              reference's (the script asserts both)
There is no CPU fallback: without a CUDA device the encoder cannot be created and the script fails.

    python tools/bench_renditions.py [--n 16] [--reps 3] [--prog-reps 1] [--sets no_restart,restart_1,progressive]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

LADDER = [((1, 1), ["-quality", "80", "-sample", "2x2"]), ((1, 2), ["-quality", "80", "-sample", "2x2"]),
          ((1, 4), ["-quality", "75", "-sample", "2x2"]), ((1, 8), ["-quality", "70", "-sample", "2x2"])]
SETS = {"no_restart": ["-revert", "-quality", "90", "-sample", "2x2"],
        "restart_1": ["-revert", "-quality", "90", "-sample", "2x2", "-restart", "1"],
        "progressive": ["-quality", "90", "-sample", "2x2"]}        # mozjpeg's default profile: progressive, scan search


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    f = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")] if r.stdout.strip() else []
    return {"card": f[0], "power_limit": f[1], "sm_clock": f[2]} if len(f) == 3 else {"card": "unknown"}


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2], ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--prog-reps", type=int, default=1, help="timed runs of the progressive set (its decode takes about a second per image)")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--sets", default="no_restart,restart_1,progressive")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_renditions.py needs a CUDA device")
    import mozjpeg_b200 as mj
    import decompress_options_cases as DO
    import recompress_cases as R
    from mozjpeg_b200 import djpeg
    from oracle import oracle as O
    W, H, N = 3840, 2160, a.n
    enc = mj.Encoder(0)
    pool = ThreadPoolExecutor(a.threads)
    for sset in a.sets.split(","):
        sw = SETS[sset]
        reps = a.prog_reps if sset == "progressive" else a.reps
        enc.set_progressive_decode(sset == "progressive")
        ps = mj.params_from_switches(sw, W, H, 3)
        srcs = list(pool.map(lambda i: O.oracle_encode(ps, O.synth_image(3000 + i, W, H)).jpeg, range(N)))
        base = dict(set=sset, images=N, width=W, height=H, source_switches=sw, source_mb=round(sum(map(len, srcs)) / 1e6, 1),
                    rungs=[f"{s[0]}/{s[1]} {' '.join(q)}" for s, q in LADDER])
        rungs = [(mj.params_for_jpeg_input(q, srcs[0], scale=s), dict(scale=s)) for s, q in LADDER]
        # the ladder (its first run warms up) and the separate calls
        out = enc.recompress_renditions(srcs, rungs)
        t, ts = timed(lambda: enc.recompress_renditions(srcs, rungs), reps)
        stages = {k: round(v / N, 4) for k, v in enc.stage_times().items()}
        print(json.dumps(dict(card(), **base, what="ladder", images_per_s=round(N / t, 2), ms_min=round(min(ts) * 1e3, 1), ms_median=round(t * 1e3, 1),
                              reps=len(ts), stage_ms_per_image=stages)), flush=True)
        sep = [enc.recompress(p, srcs, **kw) for p, kw in rungs]
        t, ts = timed(lambda: [enc.recompress(p, srcs, **kw) for p, kw in rungs], reps)
        print(json.dumps(dict(card(), **base, what="separate", calls=len(rungs), images_per_s=round(N / t, 2), ms_min=round(min(ts) * 1e3, 1),
                              ms_median=round(t * 1e3, 1), reps=len(ts))), flush=True)
        same = sum(o == s for r in range(len(rungs)) for o, s in zip(out[r], sep[r]))
        check = dict(base, what="check", identical_to_separate_calls=f"{same}/{N * len(rungs)}")
        if DO.have_reference() and R.have_reference():
            def ref(job):
                r, i = job
                (num, den), q = LADDER[r]
                px, _, msg = DO.ref_decompress(srcs[i], (num, den, 0, 1, -1))
                if px is None:
                    raise RuntimeError(msg)
                return R.insert_markers(R.ref_cjpeg(djpeg.ppm_bytes(px), q), R.copied_markers(srcs[i], rungs[r][0]))
            jobs = [(r, i) for r in range(len(rungs)) for i in range(N)]
            t0 = time.perf_counter()
            want = list(pool.map(ref, jobs))
            t = time.perf_counter() - t0
            print(json.dumps(dict(card(), **base, what="ref", host_threads=a.threads, images_per_s=round(N / t, 2), ms=round(t * 1e3, 1), reps=1)), flush=True)
            ref_same = sum(out[r][i] == w for (r, i), w in zip(jobs, want))
            check["identical_to_reference"] = f"{ref_same}/{N * len(rungs)}"
        print(json.dumps(check), flush=True)
        assert same == N * len(rungs), f"{N * len(rungs) - same} ladder files differ from the separate calls"
        if "identical_to_reference" in check:
            assert ref_same == N * len(rungs), f"{N * len(rungs) - ref_same} ladder files differ from the reference"
    enc.close()
    pool.shutdown()


if __name__ == "__main__":
    main()
