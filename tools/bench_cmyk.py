"""Decompressing and recompressing CMYK and YCCK JPEG files on the device (the `cmyk` decompress option), on N seeded
3840x2160 sources written at quality 90 by the CPU oracle (tests/colorspace_cases.py, which matches the reference's
encoder): YCCK 4:2:0 (2x2, 1x1, 1x1, 2x2) and CMYK 4:4:4, each without restarts and with a restart every MCU.  Prints
JSON lines, each carrying the card's name, power limit and SM clocks read in this run:
  decompress : Encoder.decompress_ptr with cmyk=True, pixels left in HBM: the stage times per image (dec_*, idct,
               upsample_color, which here is k_upsample_opts<4>) and, for k_upsample_opts<4>, the bytes the algorithm
               needs (one read of each sample plane, 4 bytes written per pixel) over the kernel time, against the data
               sheet's 3.35 TB/s
  recompress : cjpeg -quality 75 end to end, host file bytes to host file bytes: the device (Encoder.recompress) and the
               reference's cjpeg in.jpg on the host threads, where oracle/_ref is available; the first and the last
               device output are compared byte for byte with the reference's, or with the CPU oracle's encode of the
               decoded pixels where the reference is absent.
There is no CPU fallback: without a CUDA device the script fails.

    python tools/bench_cmyk.py [--n 16] [--reps 5] [--sets ycck420,ycck420_restart_1,cmyk444,cmyk444_restart_1]
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
SETS = {"ycck420": ("420", 5, 0), "ycck420_restart_1": ("420", 5, 1), "cmyk444": ("444", 4, 0), "cmyk444_restart_1": ("444", 4, 1)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"card": r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown"}


def spread(ts):
    ts = sorted(ts)
    return {"ms_min": round(ts[0] * 1e3, 2), "ms_median": round(ts[len(ts) // 2] * 1e3, 2), "ms_max": round(ts[-1] * 1e3, 2), "reps": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--sets", default=",".join(SETS))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_cmyk.py needs a CUDA device")
    import mozjpeg_b200 as mj
    import colorspace_cases as CS
    import recompress_cases as R
    W, H, N = 3840, 2160, a.n
    enc = mj.Encoder(0)
    pool = ThreadPoolExecutor(a.threads)
    rsw = ["-quality", "75"]
    for sset in a.sets.split(","):
        samp, cs, restart = SETS[sset]
        ps = mj.tj3_params(W, H, quality=90, subsamp=samp, cmyk=True, colorspace=cs)
        ps.restart_interval = restart
        srcs = list(pool.map(lambda i: CS.oracle_encode(ps, CS.cmyk_image(2000 + i, W, H)).jpeg, range(N)))
        base = dict(card(), set=sset, images=N, width=W, height=H, source_mb=round(sum(map(len, srcs)) / 1e6, 1))
        # (a) decompress, pixels left in HBM
        buf = torch.empty((N, H, W * 4), dtype=torch.uint8, device="cuda")
        st = []
        for _ in range(1 + a.reps):                                     # the first run warms up
            enc.decompress_ptr(srcs, buf.data_ptr(), W * 4, H * W * 4, cmyk=True)
            st.append(enc.stage_times())
        st = st[1:]
        stages = {k: round(sorted(s[k] for s in st)[len(st) // 2] / N, 4) for k in st[0]}          # median over the runs, ms per image
        # one read of each sample plane (Y and K full size, Cb and Cr at a quarter for 4:2:0), 4 bytes out per pixel
        planes = W * H * (2 + 2 * (0.25 if samp == "420" else 1.0))
        up_b = planes + W * H * 4
        print(json.dumps(dict(base, what="decompress", stage_ms_per_image=stages, total_ms_per_image=round(sum(stages.values()), 4),
                              upsample4_algorithmic_gbs=round(up_b / stages["upsample_color"] / 1e6, 1),
                              upsample4_share_of_hbm_peak=round(up_b / (stages["upsample_color"] * 1e-3) / HBM_PEAK, 3))), flush=True)
        # (b) recompress end to end against the reference
        p = mj.params_for_jpeg_input(rsw, srcs[0], cmyk=True)
        host_px = buf.cpu()
        del buf
        out = enc.recompress(p, srcs, cmyk=True)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter(); enc.recompress(p, srcs, cmyk=True); ts.append(time.perf_counter() - t0)
        t = sorted(ts)[len(ts) // 2]
        print(json.dumps(dict(base, what="recompress", route="device", switches=rsw, images_per_s=round(N / t, 1), mpixels_per_s=round(N * W * H / t / 1e6, 1),
                              **spread(ts))), flush=True)
        if R.have_reference():
            t0 = time.perf_counter()
            want = list(pool.map(lambda s: R.ref_cjpeg(s, rsw), srcs))
            t = time.perf_counter() - t0
            print(json.dumps(dict(base, what="recompress", route="ref", switches=rsw, host_threads=a.threads, images_per_s=round(N / t, 1),
                                  mpixels_per_s=round(N * W * H / t / 1e6, 1), ms_min=round(t * 1e3, 2), reps=1)), flush=True)
            check = "reference cjpeg"
        else:
            from oracle import oracle as O
            want = {i: R.insert_markers(O.oracle_encode(p, host_px[i].numpy().reshape(H, W, 4)).jpeg, R.copied_markers(srcs[i], p)) for i in (0, N - 1)}
            check = "CPU oracle encode of the decoded pixels (reference build absent)"
        for i in (0, N - 1):
            assert out[i] == want[i], f"image {i}: device output differs from the {check}"
        print(json.dumps(dict(base, what="check", first_and_last_output_byte_identical_to=check)), flush=True)
    enc.close()
    pool.shutdown()


if __name__ == "__main__":
    main()
