"""Recompressing JPEG files on the device, on N seeded 3840x2160 4:2:0 sources written with the reference's settings
-revert -quality 90 (by the CPU oracle, bit-identical to the reference's cjpeg), once without restarts and once with
-restart 1 (the two source sets of tools/bench_transcode.py).  Prints JSON lines, each carrying the card's name, SM
count and power limit read in this run:
  decompress : Encoder.decompress_ptr, pixels left in HBM: the stage times per image (dec_*, idct, upsample_color)
               and, for the two new kernels, the bytes the algorithm needs (coefficients in + samples out; samples in +
               pixels out) over the kernel time, against the data sheet's 3.35 TB/s
  recompress : cjpeg -baseline -quality 75 -sample 2x2 end to end, host file bytes to host file bytes, by three routes:
               device (Encoder.recompress), pixels (Encoder.encode_batch_ptr from pinned host pixels of the same images:
               the route when something else has decoded them) and ref (the reference's cjpeg in.jpg on the host threads,
               where oracle/_ref is available); the first and the last device output are compared byte for byte with
               the reference's, or with the CPU oracle's encode of the decoded pixels where the reference is absent.
There is no CPU fallback: without a CUDA device the encoder cannot be created and the script fails.

    python tools/bench_recompress.py [--n 32] [--reps 5] [--sets no_restart,restart_1]
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
    import torch
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"card": r.stdout.strip().splitlines()[0] if r.stdout.strip() else "unknown", "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def spread(ts):
    ts = sorted(ts)
    return {"ms_min": round(ts[0] * 1e3, 2), "ms_median": round(ts[len(ts) // 2] * 1e3, 2), "ms_max": round(ts[-1] * 1e3, 2), "reps": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--sets", default="no_restart,restart_1")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_recompress.py needs a CUDA device")
    import mozjpeg_b200 as mj
    import recompress_cases as R
    from oracle import oracle as O
    W, H, N = 3840, 2160, a.n
    hw = card()
    enc = mj.Encoder(0)
    pool = ThreadPoolExecutor(a.threads)
    rsw = ["-baseline", "-quality", "75", "-sample", "2x2"]
    for sset, sw in (("no_restart", ["-revert", "-quality", "90"]), ("restart_1", ["-revert", "-quality", "90", "-restart", "1"])):
        if sset not in a.sets.split(","):
            continue
        ps = mj.params_from_switches(sw, W, H, 3)
        srcs = list(pool.map(lambda i: O.oracle_encode(ps, O.synth_image(1000 + i, W, H)).jpeg, range(N)))
        base = dict(hw, set=sset, images=N, width=W, height=H, source_mb=round(sum(map(len, srcs)) / 1e6, 1))
        # (a) decompress, pixels left in HBM
        buf = torch.empty((N, H, W * 3), dtype=torch.uint8, device="cuda")
        st = []
        for _ in range(1 + a.reps):                                     # the first run warms up
            enc.decompress_ptr(srcs, buf.data_ptr(), W * 3, H * W * 3)
            st.append(enc.stage_times())
        st = st[1:]
        stages = {k: round(sorted(s[k] for s in st)[len(st) // 2] / N, 4) for k in st[0]}          # median over the runs, ms per image
        blocks = (W // 8) * (H // 8) + 2 * (W // 16) * (H // 16)
        idct_b, up_b = blocks * (128 + 64), blocks * 64 + W * H * 3
        print(json.dumps(dict(base, what="decompress", stage_ms_per_image=stages, total_ms_per_image=round(sum(stages.values()), 4),
                              idct_algorithmic_gbs=round(idct_b / stages["idct"] / 1e6, 1), idct_share_of_hbm_peak=round(idct_b / (stages["idct"] * 1e-3) / HBM_PEAK, 3),
                              upsample_color_algorithmic_gbs=round(up_b / stages["upsample_color"] / 1e6, 1),
                              upsample_color_share_of_hbm_peak=round(up_b / (stages["upsample_color"] * 1e-3) / HBM_PEAK, 3))), flush=True)
        # (b) recompress end to end against the pixel route and the reference
        p = mj.params_for_jpeg_input(rsw, srcs[0])
        host_px = buf.cpu().pin_memory()
        del buf

        def device():
            return enc.recompress(p, srcs)

        def pixels():
            enc.encode_batch_ptr(p, host_px.data_ptr(), False, W * 3, H * W * 3, N)
            return [enc.get_output(i) for i in range(N)]

        outs = {}
        for name, fn in (("device", device), ("pixels", pixels)):
            outs[name] = fn()
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
            t = sorted(ts)[len(ts) // 2]
            print(json.dumps(dict(base, what="recompress", route=name, switches=rsw, images_per_s=round(N / t, 1), mpixels_per_s=round(N * W * H / t / 1e6, 1), **spread(ts))), flush=True)
        assert outs["device"] == outs["pixels"], "recompress differs from the encode of the decoded pixels"
        # (c) the reference
        if R.have_reference():
            t0 = time.perf_counter()
            want = list(pool.map(lambda s: R.ref_cjpeg(s, rsw), srcs))
            t = time.perf_counter() - t0
            print(json.dumps(dict(base, what="recompress", route="ref", switches=rsw, host_threads=a.threads, images_per_s=round(N / t, 1),
                                  mpixels_per_s=round(N * W * H / t / 1e6, 1), ms_min=round(t * 1e3, 2), reps=1)), flush=True)
            check = "reference cjpeg"
        else:
            want = {i: O.oracle_encode(p, host_px[i].numpy().reshape(H, W, 3)).jpeg for i in (0, N - 1)}
            check = "CPU oracle encode of the decoded pixels (reference build absent)"
        for i in (0, N - 1):
            assert outs["device"][i] == want[i], f"image {i}: device output differs from the {check}"
        print(json.dumps(dict(base, what="check", first_and_last_output_byte_identical_to=check)), flush=True)
    enc.close()
    pool.shutdown()


if __name__ == "__main__":
    main()
