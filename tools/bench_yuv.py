"""YUV encoding (tj3EncodeYUVPlanes8 on the device, k_encode_yuv) throughput, one JSON line per workload:
  * N x 3840x2160 RGB to 4:2:0 and to 4:4:4, pixels and planes in HBM: CUDA events around back-to-back batches on the
    caller's stream for at least --seconds after a warm-up, and the kernel's own event time (b200jpeg_last_stage_times);
  * the same batch from pinned host memory to pinned host planes, end to end (host clock around the synchronous call);
  * the reference's tj3EncodeYUVPlanes8 (oracle/_ref/libturbojpeg_ref.so) on every host thread, as the CPU arm.
Each line holds GP/s, the algorithmic bytes (W*H*C read + sum of pw*ph written) over kernel time as a share of the H100
SXM datasheet's 3.35 TB/s, whether the first and last images' planes equal the reference's, and the card's name and
power limit read in the same run.

    python tools/bench_yuv.py [--images 256] [--seconds 1.0] [--cpu-images 64]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM_TBPS = 3.35          # H100 SXM datasheet HBM3 bandwidth


def card():
    import torch
    prop = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"name": prop.name, "sms": prop.multi_processor_count, "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def make_batch(n, h, w):
    """Seeded RGB content generated on the device: gradients plus noise."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(11)
    yy = torch.arange(h, device="cuda", dtype=torch.int32).view(h, 1, 1)
    xx = torch.arange(w, device="cuda", dtype=torch.int32).view(1, w, 1)
    cc = torch.arange(3, device="cuda", dtype=torch.int32).view(1, 1, 3)
    base = (xx * (3 + cc) + yy * (2 + 5 * cc)) % 256
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
    for i in range(n):
        noise = torch.randint(-24, 25, (h, w, 3), generator=g, device="cuda", dtype=torch.int32)
        out[i] = (base + i * 7 + noise).clamp(0, 255).to(torch.uint8)
    return out


def run(enc, ss, pix, seconds, cpu_images):
    import torch
    import mozjpeg_b200 as mj
    import yuv_cases as Y
    n, h, w, c = pix.shape
    p = mj.tj3_params(w, h, subsamp=ss, pixel_format="RGB")
    geo = [mj.yuv_plane_dims(p, ci) for ci in range(p.num_components)]
    planes = [torch.empty((n, ph, pw), dtype=torch.uint8, device="cuda") for pw, ph in geo]
    pitch, stride = [pw for pw, _ in geo], [pw * ph for pw, ph in geo]
    ptrs = [t.data_ptr() for t in planes]
    stream = torch.cuda.current_stream()
    enc.set_stream(stream.cuda_stream)

    def call():
        enc.encode_yuv_batch_ptr(p, pix.data_ptr(), True, w * c, h * w * c, ptrs, True, pitch, stride, n)

    call(); call()                                           # warm-up
    torch.cuda.synchronize()
    kernel_ms = enc.stage_times()["encode_yuv"]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps, t_start = 0, time.perf_counter()
    e0.record(stream)
    while True:
        call(); reps += 1
        if reps % 4 == 0:
            torch.cuda.synchronize()
            if time.perf_counter() - t_start >= seconds:
                break
    e1.record(stream)
    torch.cuda.synchronize()
    dev_ms = e0.elapsed_time(e1) / reps
    kernels = []
    for _ in range(5):
        call()
        kernels.append(enc.stage_times()["encode_yuv"])
    kernel_ms = float(np.median(kernels))
    # parity: first and last image against the reference
    ref = Y.RefTJ()
    parity = True
    for i in (0, n - 1):
        img = pix[i].cpu().numpy()
        want, err = ref.encode_planes(img, "RGB", ss)
        got = [t[i].cpu().numpy() for t in planes]
        parity = parity and err is None and all(np.array_equal(a, b) for a, b in zip(want, got))
    print("bench_yuv: device-resident done, pinned host arm", file=sys.stderr, flush=True)
    # end to end from and to pinned host memory
    hpix = torch.empty(pix.shape, dtype=torch.uint8, pin_memory=True)
    hpix.copy_(pix)
    hplanes = [torch.empty(t.shape, dtype=torch.uint8, pin_memory=True) for t in planes]
    hptrs = [t.data_ptr() for t in hplanes]

    def call_host():
        enc.encode_yuv_batch_ptr(p, hpix.data_ptr(), False, w * c, h * w * c, hptrs, False, pitch, stride, n)
    call_host()
    host_ms = []
    for _ in range(3):
        t0 = time.perf_counter(); call_host(); host_ms.append((time.perf_counter() - t0) * 1e3)
    host_stages = enc.stage_times()
    host_parity = all(torch.equal(a.cpu(), b) for a, b in zip(planes, hplanes))
    del hpix, hplanes
    # the reference on every host thread
    threads = os.cpu_count() or 1
    k = min(cpu_images, n)
    imgs = pix[:k].cpu().numpy()
    local, handles = threading.local(), []              # a TurboJPEG handle belongs to one thread

    def ref_one(i):
        if not hasattr(local, "tj"):
            local.tj = Y.RefTJ(); handles.append(local.tj)
        local.tj.encode_planes(imgs[i], "RGB", ss)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(ref_one, range(k)))
    ref_s = time.perf_counter() - t0
    for r in handles:
        r.close()
    ref.close()
    gp = n * w * h / 1e9
    nbytes = n * (w * h * c + sum(pw * ph for pw, ph in geo))
    return {"workload": f"rgb_to_{ss}", "images": n, "width": w, "height": h,
            "device_resident": {"ms_per_batch": dev_ms, "gpps": gp / (dev_ms / 1e3), "batches_timed": reps,
                                "kernel_ms": kernel_ms, "kernel_gpps": gp / (kernel_ms / 1e3),
                                "algorithmic_bytes": nbytes, "kernel_tbps": nbytes / (kernel_ms / 1e3) / 1e12,
                                "share_of_datasheet_hbm": nbytes / (kernel_ms / 1e3) / 1e12 / HBM_TBPS},
            "pinned_host_end_to_end": {"ms_per_batch_best": min(host_ms), "ms_per_batch_median": float(np.median(host_ms)),
                                       "gpps": gp / (min(host_ms) / 1e3), "stage_ms": host_stages, "equal_to_device_resident": host_parity},
            "parity_first_last_vs_reference": parity,
            "reference_host_threads": threads, "reference_images": k, "reference_host_gpps": k * w * h / 1e9 / ref_s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--cpu-images", type=int, default=64)
    a = ap.parse_args()
    import torch
    import mozjpeg_b200 as mj
    if not torch.cuda.is_available():
        raise SystemExit("bench_yuv: no CUDA device")
    info = card()
    print("bench_yuv: generating", a.images, "images", file=sys.stderr, flush=True)
    pix = make_batch(a.images, 2160, 3840)
    enc = mj.Encoder(0)
    for ss in ("420", "444"):
        print("bench_yuv:", ss, file=sys.stderr, flush=True)
        r = run(enc, ss, pix, a.seconds, a.cpu_images)
        r["card"] = info
        print(json.dumps(r), flush=True)
    enc.close()


if __name__ == "__main__":
    main()
