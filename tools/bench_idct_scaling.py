"""Decompressing at every TurboJPEG scaling factor on the device (all_scales), on N seeded 3840x2160 4:2:0 sources written
with -revert -quality 90 -sample 2x2 by the CPU oracle (the source set of tools/bench_yuv_decode.py), once without
restarts and once with -restart 1.  Prints JSON lines, each carrying the card's name, power limit and SM clock read in
this run:
  pixels     : per factor, Encoder.decompress_ptr to RGB pixels left in HBM: images/s and the stage times per image
               (dec_*, idct, upsample_color); for the IDCT the bytes it needs (128 coefficient bytes read a block, the
               ssize * ssize samples written) over its stage time, against the data sheet's 3.35 TB/s
  host       : the same to host pixels (Encoder.decompress)
  yuv        : per factor, Encoder.decompress_yuv_ptr into planes left in HBM: images/s and the IDCT stage
  ref_pixels : the reference library's decode at the factor (tests/refdecopt.c, djpeg's path) on --threads host threads
  ref_yuv    : the reference's tj3DecompressToYUVPlanes8 on --threads host threads
  ratio      : end-to-end time of 3/4 and 7/8 against 1/1, and 3/8 against 1/2, into HBM
With --old only the stage totals of the old scales (1/8 .. 1/1, pixels and YUV planes) are printed, for comparing two
builds of the library (B200JPEG_LIB_VARIANT) run alternately.  There is no CPU fallback: without a CUDA device the
script fails.

    python tools/bench_idct_scaling.py [--n 16] [--reps 3] [--threads 16] [--sets no_restart,restart_1] [--old]
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
HBM_PEAK = 3.35e12            # H100 SXM data sheet, bytes/s
FACTORS = [(1, 8), (1, 4), (3, 8), (1, 2), (5, 8), (3, 4), (7, 8), (1, 1), (9, 8), (5, 4), (11, 8), (3, 2), (13, 8), (7, 4), (15, 8), (2, 1)]
OLD = [(1, 8), (1, 4), (1, 2), (1, 1)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"card": r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown", "lib": os.environ.get("B200JPEG_LIB_VARIANT") or "tree"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--sets", default="no_restart,restart_1")
    ap.add_argument("--old", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_idct_scaling.py needs a CUDA device")
    import mozjpeg_b200 as mj
    import decompress_options_cases as D
    import yuv_decode_cases as Y
    from oracle import oracle as O
    W, H, N = 3840, 2160, a.n
    enc = mj.Encoder(0)
    sets = {"no_restart": ["-revert", "-quality", "90", "-sample", "2x2"], "restart_1": ["-revert", "-quality", "90", "-sample", "2x2", "-restart", "1"]}
    for sset in a.sets.split(","):
        p = mj.params_from_switches(sets[sset], W, H, 3)
        srcs = [O.oracle_encode(p, O.synth_image(900 + i, W, H)).jpeg for i in range(N)]
        info = mj._parse_first(srcs)
        base = {**card(), "set": sset, "images": N, "size": f"{W}x{H}"}

        def timed(fn):
            fn()
            torch.cuda.synchronize()
            ts, stages = [], {}
            for _ in range(a.reps):
                t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
                for k, v in enc.stage_times().items():
                    stages[k] = stages.get(k, 0.0) + v / a.reps
            return sorted(ts)[len(ts) // 2], {k: round(v / N, 3) for k, v in stages.items()}

        def kw(f):
            return dict(scale=f) if a.old else dict(scale=f, all_scales=True)

        e2e = {}
        for f in (OLD if a.old else FACTORS):
            ow, oh, comps = D.plan(info, f, True)
            blocks = [-(-W * info.h_samp_factor[c] // (2 * 8)) * -(-H * info.v_samp_factor[c] // (2 * 8)) for c in range(3)]
            idct_bytes = N * sum(b * 128 + b * c[0] * c[0] for b, c in zip(blocks, comps))
            pix = torch.empty(N * ow * oh * 3, dtype=torch.uint8, device="cuda")
            t, st = timed(lambda: enc.decompress_ptr(srcs, pix.data_ptr(), ow * 3, ow * oh * 3, **kw(f)))
            e2e[f] = t
            idct_s = st.get("idct", 0.0) * N / 1e3
            print(json.dumps({**base, "kind": "pixels", "scale": f"{f[0]}/{f[1]}", "ssize": [c[0] for c in comps], "images_per_s": round(N / t, 1),
                              "ms_per_image": round(t * 1e3 / N, 3), "stage_ms_per_image": st, "idct_bytes": idct_bytes,
                              "idct_GBps": round(idct_bytes / idct_s / 1e9, 1) if idct_s else None,
                              "idct_share_of_3.35TBps": round(idct_bytes / idct_s / HBM_PEAK, 3) if idct_s else None}), flush=True)
            del pix
            if not a.old:
                t, st = timed(lambda: enc.decompress(srcs, **kw(f)))
                print(json.dumps({**base, "kind": "host", "scale": f"{f[0]}/{f[1]}", "images_per_s": round(N / t, 1), "stage_ms_per_image": st}), flush=True)
            _, plan = Y.plan(info, f)
            dims = [(pw, ph) for pw, ph, _, _ in plan]
            k = 8 * f[0] // f[1]
            ybytes = N * sum((iw // k) * (ih // k) * 128 + min(iw, pw) * min(ih, ph) for pw, ph, iw, ih in plan)
            dev = [torch.empty(N * pw * ph, dtype=torch.uint8, device="cuda") for pw, ph in dims]
            t, st = timed(lambda: enc.decompress_yuv_ptr(srcs, [d.data_ptr() for d in dev], [pw for pw, _ in dims], [pw * ph for pw, ph in dims], **kw(f)))
            idct_s = st.get("idct", 0.0) * N / 1e3
            print(json.dumps({**base, "kind": "yuv", "scale": f"{f[0]}/{f[1]}", "images_per_s": round(N / t, 1), "stage_ms_per_image": st,
                              "idct_GBps": round(ybytes / idct_s / 1e9, 1) if idct_s else None,
                              "idct_share_of_3.35TBps": round(ybytes / idct_s / HBM_PEAK, 3) if idct_s else None}), flush=True)
            del dev
        if a.old:
            continue
        print(json.dumps({**base, "kind": "ratio", "3/4_over_1/1": round(e2e[(3, 4)] / e2e[(1, 1)], 3), "7/8_over_1/1": round(e2e[(7, 8)] / e2e[(1, 1)], 3),
                          "3/8_over_1/2": round(e2e[(3, 8)] / e2e[(1, 2)], 3)}), flush=True)
        if D.have_reference() and os.path.exists(Y.REF_TJ):
            pool = ThreadPoolExecutor(a.threads)
            refs = [Y.RefTJ() for _ in range(a.threads)]
            for f in FACTORS:
                for kind, one in (("ref_pixels", lambda i: D.ref_decompress(srcs[i], (f[0], f[1], 0, 1, -1))),
                                  ("ref_yuv", lambda i: refs[i % a.threads].decompress_planes(srcs[i], f, "int"))):
                    t0 = time.perf_counter(); list(pool.map(one, range(N))); t = time.perf_counter() - t0
                    print(json.dumps({**base, "kind": kind, "scale": f"{f[0]}/{f[1]}", "threads": a.threads, "images_per_s": round(N / t, 1)}), flush=True)
            for r in refs:
                r.close()
    enc.close()


if __name__ == "__main__":
    main()
