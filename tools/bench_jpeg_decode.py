"""JPEG files to HD crops: PIL decode on the host against decode_jpeg_batch on the GPU, end to end, plus the decoder's kernel times.

    python tools/bench_jpeg_decode.py [--e2e-reps 10] [--out result.json] [--trace-dir DIR]

Workload: BASELINE configs[3]'s HD batch (32 images, sizes seeded as in bench.py, patch_num 9), seeded smooth images with mild noise,
encoded by Pillow at quality 90, 4:2:0 (Pillow's defaults otherwise: baseline, no restart markers).  Prints one JSON line.

  end to end, each path ending in a device synchronise (host clock), A and B alternated, their crops asserted bit-equal
    (A)  PIL decode (Image.open(...).convert('RGB')) on a 16-thread host pool into pinned uint8, upload, hd_preprocess_batch(bf16)
    (B)  decode_jpeg_batch from the files' bytes (host plan, one upload of the scans and tables, four launches), hd_preprocess_batch(bf16)
    (B0) decode_jpeg_batch alone
  kernel times per stage from torch.profiler (CUDA activities) in a run of its own, averaged over the profiled calls, and the
  synchronisation rounds of every file.  Writes nothing but --out (and the trace under --trace-dir when given).
"""
from __future__ import annotations

import argparse
import io
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_hd_preprocess import card  # noqa: E402


def workload():
    g = torch.Generator().manual_seed(0)                       # bench.py's configs[3] sizes
    hs = torch.randint(224, 1345, (32,), generator=g).tolist()
    ws = torch.randint(224, 1345, (32,), generator=g).tolist()
    rng = np.random.default_rng(1234)
    files = []
    for h, w in zip(hs, ws):
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        base = np.stack([128 + 100 * np.sin(xx / 37 + c) * np.cos(yy / 53 - c) for c in range(3)], 2)
        a = np.clip(base + rng.normal(0, 6, (h, w, 3)), 0, 255).astype(np.uint8)
        b = io.BytesIO()
        Image.fromarray(a).save(b, "JPEG", quality=90, subsampling=2)
        files.append(b.getvalue())
    return hs, ws, files


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--e2e-reps", type=int, default=10)
    ap.add_argument("--profile-calls", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-dir", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg_decode: needs a CUDA device (there is no CPU measurement)")
    from tokenpacker_b200 import decode_jpeg_batch, hd_preprocess_batch
    dev = torch.device("cuda", torch.cuda.current_device())
    hs, ws, files = workload()
    pinned = [torch.empty((h, w, 3), dtype=torch.uint8).pin_memory() for h, w in zip(hs, ws)]
    pool = ThreadPoolExecutor(16)

    def pil_into(i):
        pinned[i].numpy()[...] = np.asarray(Image.open(io.BytesIO(files[i])).convert("RGB"))

    def path_a():
        list(pool.map(pil_into, range(len(files))))
        imgs = [p.to(dev, non_blocking=True) for p in pinned]
        out, _, _ = hd_preprocess_batch(imgs, 9, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        return out

    def path_b():
        out, _, _ = hd_preprocess_batch(decode_jpeg_batch(files, dev), 9, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        return out

    def path_b0():
        decode_jpeg_batch(files, dev, return_status=True)
        torch.cuda.synchronize()

    a, b = path_a(), path_b()                                   # warm-up, and the bit check
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "A and B differ"
    n_crops = a.shape[0]
    del a, b
    e2e = {"A_pil_pool16": [], "B_gpu_decode": [], "B0_gpu_decode_only": []}
    for _ in range(args.e2e_reps):
        for k, fn in (("A_pil_pool16", path_a), ("B_gpu_decode", path_b), ("B0_gpu_decode_only", path_b0)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            e2e[k].append((time.perf_counter() - t0) * 1e3)
    # PIL on one core, for the per-image cost the host pays without a pool
    t0 = time.perf_counter()
    for f in files:
        Image.open(io.BytesIO(f)).convert("RGB")
    pil_one_core_ms = (time.perf_counter() - t0) * 1e3

    _, status = decode_jpeg_batch(files, dev, return_status=True)
    st = status.cpu().numpy()
    assert (st[:, 0] == 0).all()

    # kernel times, a run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.profile_calls):
            decode_jpeg_batch(files, dev, return_status=True)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if "jpeg" in e.key:
            name = e.key.split("(")[0].split("::")[-1]
            kern[name] = {"calls": e.count, "avg_us": e.device_time_total / max(e.count, 1)}
    if args.trace_dir:
        os.makedirs(args.trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace_dir, "jpeg_decode.pt.trace.json"))

    rec = {"what": "32 JPEG files (configs[3] sizes 224..1344, q90 4:2:0) -> patch_num 9 -> %d bf16 crops" % n_crops, "card": card(dev),
           "jpeg_bytes": sum(len(f) for f in files), "decoded_bytes": sum(h * w * 3 for h, w in zip(hs, ws)),
           "e2e_ms_median": {k: statistics.median(v) for k, v in e2e.items()}, "e2e_ms_min": {k: min(v) for k, v in e2e.items()},
           "e2e_bits_equal": True, "pil_one_core_ms_batch": pil_one_core_ms, "kernel_us": kern,
           "sync_rounds": st[:, 1].tolist(), "subsequences": st[:, 2].tolist(), "host_threads_pool": 16, "cpu_count": os.cpu_count()}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
