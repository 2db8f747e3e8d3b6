"""Decompressing to YUV planes on the device (Encoder.decompress_yuv, tj3DecompressToYUVPlanes8) on N seeded 3840x2160
4:2:0 sources written with -revert -quality 90 -sample 2x2 by the CPU oracle, once without restarts and once with
-restart 1.  Prints JSON lines, each carrying the card's name, power limit and SM clock read in this run:
  yuv_device : planes left in HBM (Encoder.decompress_yuv_ptr), per scale 1/1 and 1/2 x dct int / fast: images/s and
               the stage times per image (dec_*, idct); for the IDCT-to-plane stage the bytes the algorithm needs (128
               coefficient bytes read a block, the k * k samples written) over its time, against 3.35 TB/s
  yuv_host   : the same into host planes (one compact staging buffer, one copy per plane and image)
  pixels     : Encoder.decompress_ptr to RGB pixels in HBM on the same sources, for comparison
  ref        : the reference's tj3DecompressToYUVPlanes8 (oracle/_ref/libturbojpeg_ref.so) on --threads host threads,
               one handle per thread, where that library is present
  check      : the device planes equal the reference's (defined samples) for the first image
  decode_yuv : Encoder.decode_yuv_ptr of 3840x2160 4:2:0 planes to RGB pixels, both in HBM: images/s, the
               yuv_to_pixels stage and its bytes (12.4 MB of planes read, 24.9 MB of pixels written per image) over its
               time against 3.35 TB/s
There is no CPU fallback: without a CUDA device the script fails.

    python tools/bench_yuv_decode.py [--n 16] [--reps 5] [--threads 16]
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"card": r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=16)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_yuv_decode.py needs a CUDA device")
    import mozjpeg_b200 as mj
    import yuv_decode_cases as Y
    from oracle import oracle as O
    W, H, N = 3840, 2160, a.n
    enc = mj.Encoder(0)
    for sset, sw in (("no_restart", ["-revert", "-quality", "90", "-sample", "2x2"]), ("restart_1", ["-revert", "-quality", "90", "-sample", "2x2", "-restart", "1"])):
        p = mj.params_from_switches(sw, W, H, 3)
        srcs = [O.oracle_encode(p, O.synth_image(900 + i, W, H)).jpeg for i in range(N)]
        info = mj._parse_first(srcs)
        base = {**card(), "set": sset, "images": N, "size": f"{W}x{H}", "src_mb": round(sum(map(len, srcs)) / 1e6, 2)}

        def timed(fn):
            fn()
            torch.cuda.synchronize()
            ts, stages = [], {}
            for _ in range(a.reps):
                t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
                for k, v in enc.stage_times().items():
                    stages[k] = stages.get(k, 0.0) + v / a.reps
            t = sorted(ts)[len(ts) // 2]
            return t, {k: round(v / N, 3) for k, v in stages.items()}

        for scale in ((1, 1), (1, 2)):
            for dct in ("int", "fast"):
                _, plan = Y.plan(info, scale)
                dims = [(pw, ph) for pw, ph, _, _ in plan]
                k = 8 * scale[0] // scale[1]
                blocks = sum((iw // k) * (ih // k) for _, _, iw, ih in plan)
                idct_bytes = N * sum((iw // k) * (ih // k) * 128 + min(iw, pw) * min(ih, ph) for pw, ph, iw, ih in plan)
                dev = [torch.empty(N * pw * ph, dtype=torch.uint8, device="cuda") for pw, ph in dims]
                t, st = timed(lambda: enc.decompress_yuv_ptr(srcs, [d.data_ptr() for d in dev], [pw for pw, _ in dims],
                                                             [pw * ph for pw, ph in dims], scale=scale, dct=dct))
                idct_ms = st.get("idct", 0.0) * N
                print(json.dumps({**base, "kind": "yuv_device", "scale": f"{scale[0]}/{scale[1]}", "dct": dct, "images_per_s": round(N / t, 1),
                                  "ms_per_image": round(t * 1e3 / N, 3), "stage_ms_per_image": st, "blocks_per_image": blocks,
                                  "idct_bytes": idct_bytes, "idct_GBps": round(idct_bytes / (idct_ms / 1e3) / 1e9, 1) if idct_ms else None,
                                  "idct_share_of_3.35TBps": round(idct_bytes / (idct_ms / 1e3) / HBM_PEAK, 3) if idct_ms else None}), flush=True)
                t, st = timed(lambda: enc.decompress_yuv(srcs, scale=scale, dct=dct))
                print(json.dumps({**base, "kind": "yuv_host", "scale": f"{scale[0]}/{scale[1]}", "dct": dct, "images_per_s": round(N / t, 1),
                                  "ms_per_image": round(t * 1e3 / N, 3), "stage_ms_per_image": st,
                                  "host_bytes_per_image": sum(pw * ph for pw, ph in dims)}), flush=True)
                del dev
        pix = torch.empty(N * W * H * 3, dtype=torch.uint8, device="cuda")
        t, st = timed(lambda: enc.decompress_ptr(srcs, pix.data_ptr(), W * 3, W * H * 3))
        print(json.dumps({**base, "kind": "pixels", "scale": "1/1", "dct": "int", "images_per_s": round(N / t, 1), "ms_per_image": round(t * 1e3 / N, 3),
                          "stage_ms_per_image": st, "host_bytes_per_image": W * H * 3}), flush=True)
        del pix
        if os.path.exists(Y.REF_TJ):
            refs = [Y.RefTJ() for _ in range(a.threads)]
            pool = ThreadPoolExecutor(a.threads)
            ss, planes, err = refs[0].decompress_planes(srcs[0], (1, 1), "int")
            got = enc.decompress_yuv(srcs[:1])[0]
            _, plan = Y.plan(info, (1, 1))
            ok = err is None and all(np.array_equal(Y.defined(g, *d), Y.defined(r, *d)) for g, r, d in zip(got, planes, plan))
            print(json.dumps({**base, "kind": "check", "device_equals_reference": bool(ok)}), flush=True)
            for scale, dct in (((1, 1), "int"), ((1, 2), "fast")):
                def run():
                    list(pool.map(lambda i: refs[i % a.threads].decompress_planes(srcs[i], scale, dct), range(N)))
                run()
                ts = []
                for _ in range(a.reps):
                    t0 = time.perf_counter(); run(); ts.append(time.perf_counter() - t0)
                t = sorted(ts)[len(ts) // 2]
                print(json.dumps({**base, "kind": "ref", "scale": f"{scale[0]}/{scale[1]}", "dct": dct, "threads": a.threads,
                                  "images_per_s": round(N / t, 1), "ms_per_image": round(t * 1e3 / N, 3)}), flush=True)
            for r in refs:
                r.close()
    p = mj.tj3_params(W, H, subsamp="420", pixel_format="RGB", colorspace=3)
    dims = [mj.yuv_plane_dims(p, c) for c in range(3)]
    planes = [torch.randint(0, 256, (N * pw * ph,), dtype=torch.uint8, device="cuda") for pw, ph in dims]
    pix = torch.empty(N * W * H * 3, dtype=torch.uint8, device="cuda")
    run = lambda: enc.decode_yuv_ptr(p, [t.data_ptr() for t in planes], True, [pw for pw, _ in dims], [pw * ph for pw, ph in dims],
                                     pix.data_ptr(), True, W * 3, W * H * 3, N)
    run(); torch.cuda.synchronize()
    ts, st = [], 0.0
    for _ in range(a.reps):
        t0 = time.perf_counter(); run(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
        st += enc.stage_times()["yuv_to_pixels"] / a.reps
    t = sorted(ts)[len(ts) // 2]
    nbytes = N * (sum(pw * ph for pw, ph in dims) + W * H * 3)
    print(json.dumps({**card(), "kind": "decode_yuv", "images": N, "size": f"{W}x{H}", "subsamp": "420", "pixel_format": "RGB",
                      "images_per_s": round(N / t, 1), "yuv_to_pixels_ms_per_image": round(st / N, 4), "bytes": nbytes,
                      "GBps": round(nbytes / (st / 1e3) / 1e9, 1), "share_of_3.35TBps": round(nbytes / (st / 1e3) / HBM_PEAK, 3)}), flush=True)
    enc.close()


if __name__ == "__main__":
    main()
