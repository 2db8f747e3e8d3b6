"""Decompressing with options on the device (scale, dct_method, do_fancy_upsampling), on N seeded 3840x2160 4:2:0
sources written with -revert -quality 90 -sample 2x2 by the CPU oracle, once without restarts and once with -restart 1.
Prints JSON lines, each carrying the card's name, power limit and SM clock read in this run:
  decompress : Encoder.decompress_ptr, pixels left in HBM, for scale 1/1, 1/2, 1/4, 1/8 x dct int / fast / float x fancy
               on / off: the stage times per image (dec_*, idct, upsample_color) and, for the IDCT and the upsampling /
               colour conversion, the bytes the algorithm needs over the stage time against the data sheet's 3.35 TB/s
               (IDCT: the coefficient sectors read, 128 bytes a block, 32 for the DC-only 1x1, plus k * k samples written;
               upsample_color: the sample planes read once plus the pixels written)
  rendition  : a 1/4-scale rendition recompressed with -quality 75 -sample 2x2, host file bytes to host file bytes:
               device (Encoder.recompress with scale=(1, 4)) and ref (the reference library's scaled decode,
               tests/refdecopt.c, then the reference's cjpeg on the PPM, on the host threads, where oracle/_ref is
               available)
  check      : every device rendition byte-identical to the reference's (or, without the reference build, to the
               device encode of the device's scaled decode)
There is no CPU fallback: without a CUDA device the encoder cannot be created and the script fails.

    python tools/bench_decompress_options.py [--n 16] [--reps 5] [--sets no_restart,restart_1]
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
    ap.add_argument("--sets", default="no_restart,restart_1")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_decompress_options.py needs a CUDA device")
    import mozjpeg_b200 as mj
    import decompress_options_cases as DO
    import recompress_cases as R
    from mozjpeg_b200 import djpeg
    from oracle import oracle as O
    W, H, N = 3840, 2160, a.n
    enc = mj.Encoder(0)
    pool = ThreadPoolExecutor(a.threads)
    rsw = ["-quality", "75", "-sample", "2x2"]
    for sset, sw in (("no_restart", ["-revert", "-quality", "90", "-sample", "2x2"]), ("restart_1", ["-revert", "-quality", "90", "-sample", "2x2", "-restart", "1"])):
        if sset not in a.sets.split(","):
            continue
        ps = mj.params_from_switches(sw, W, H, 3)
        srcs = list(pool.map(lambda i: O.oracle_encode(ps, O.synth_image(2000 + i, W, H)).jpeg, range(N)))
        base = dict(set=sset, images=N, width=W, height=H, source_mb=round(sum(map(len, srcs)) / 1e6, 1))
        buf = torch.empty((N, H, W * 3), dtype=torch.uint8, device="cuda")
        lb, cb = (W // 8) * (H // 8), (W // 16) * (H // 16)          # luma and chroma blocks per image
        for scale in ((1, 1), (1, 2), (1, 4), (1, 8)):
            k = 8 // scale[1]
            for dct in ("int", "fast", "float"):
                for fancy in (True, False):
                    ow, oh = -(-W * k // 8), -(-H * k // 8)
                    st = []
                    for _ in range(1 + a.reps):                         # the first run warms up
                        enc.decompress_ptr(srcs, buf.data_ptr(), ow * 3, oh * ow * 3, scale=scale, dct=dct, fancy=fancy)
                        st.append(enc.stage_times())
                    st = st[1:]
                    stages = {s: round(sorted(t[s] for t in st)[len(st) // 2] / N, 4) for s in st[0]}
                    ck = min(8, 2 * k)                                  # chroma's DCT_scaled_size (scaled up through the IDCT)
                    idct_b = lb * ((128 if k > 1 else 32) + k * k) + 2 * cb * ((128 if ck > 1 else 32) + ck * ck)
                    up_b = lb * k * k + 2 * cb * ck * ck + ow * oh * 3
                    hw = card()
                    print(json.dumps(dict(hw, **base, what="decompress", scale=f"{scale[0]}/{scale[1]}", dct=dct, fancy=fancy, output=[ow, oh],
                                          stage_ms_per_image=stages, total_ms_per_image=round(sum(stages.values()), 4),
                                          idct_algorithmic_gbs=round(idct_b / stages["idct"] / 1e6, 1),
                                          idct_share_of_hbm_peak=round(idct_b / (stages["idct"] * 1e-3) / HBM_PEAK, 3),
                                          upsample_color_algorithmic_gbs=round(up_b / stages["upsample_color"] / 1e6, 1),
                                          upsample_color_share_of_hbm_peak=round(up_b / (stages["upsample_color"] * 1e-3) / HBM_PEAK, 3))), flush=True)
        del buf
        # the 1/4 rendition, end to end
        kw = dict(scale=(1, 4))
        p = mj.params_for_jpeg_input(rsw, srcs[0], **kw)
        out = enc.recompress(p, srcs, **kw)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter(); enc.recompress(p, srcs, **kw); ts.append(time.perf_counter() - t0)
        t = sorted(ts)[len(ts) // 2]
        print(json.dumps(dict(card(), **base, what="rendition", route="device", scale="1/4", switches=rsw, images_per_s=round(N / t, 1),
                              ms_min=round(min(ts) * 1e3, 2), ms_median=round(t * 1e3, 2), reps=len(ts))), flush=True)
        if DO.have_reference():
            def ref(s):
                px, _, msg = DO.ref_decompress(s, (1, 4, 0, 1, -1))
                return R.ref_cjpeg(djpeg.ppm_bytes(px), rsw)
            t0 = time.perf_counter()
            want = list(pool.map(ref, srcs))
            t = time.perf_counter() - t0
            print(json.dumps(dict(card(), **base, what="rendition", route="ref", scale="1/4", switches=rsw, host_threads=a.threads,
                                  images_per_s=round(N / t, 1), ms=round(t * 1e3, 2), reps=1)), flush=True)
            check = "the reference's scaled decode + cjpeg"
        else:
            px = enc.decompress(srcs, **kw)
            want = enc.encode_batch(p, px)
            check = "the device encode of the device's scaled decode (reference build absent)"
        same = sum(o == w for o, w in zip(out, want))
        print(json.dumps(dict(base, what="check", renditions_byte_identical=f"{same}/{N}", against=check)), flush=True)
        assert same == N, f"{N - same} renditions differ from {check}"
    enc.close()
    pool.shutdown()


if __name__ == "__main__":
    main()
