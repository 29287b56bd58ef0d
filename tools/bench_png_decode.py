"""PNG files to HD crops: PIL decode on the host against decode_png_batch on the GPU, end to end, per content kind, plus the decoder's
kernel times and block statistics.

    python tools/bench_png_decode.py [--e2e-reps 5] [--out result.json] [--trace-dir DIR]

Workload: BASELINE configs[3]'s HD batch (32 images, sizes seeded as in bench.py, patch_num 9) in three contents, each saved by
Pillow with its defaults (compress_level 6): document-like gray text on white ('L'), chart-like flat colour bars in an adaptive
palette ('P') and photo-like smooth RGB with mild noise ('RGB').  Prints one JSON line.

  end to end, each path ending in a device synchronise (host clock), A and B alternated, their crops asserted bit-equal
    (A)  PIL decode (Image.open(...).convert('RGB')) on a 16-thread host pool into pinned uint8, upload, hd_preprocess_batch(bf16)
    (B)  decode_png_batch from the files' bytes, hd_preprocess_batch(bf16)
    (B0) decode_png_batch alone
  kernel times per stage from torch.profiler (CUDA activities) in a run of its own, and per file the true blocks, the blocks the
  chain decoded itself and the candidate block starts.  Writes nothing but --out (and the trace under --trace-dir when given).
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


def content(kind, h, w, rng):
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "L":
        a = np.full((h, w), 250, np.uint8)
        line = (yy % 18 < 9) & (xx % 7 < 5) & (rng.random((h, w)) < 0.45) & (xx > w // 12) & (xx < w - w // 12)
        a[line] = 30
        return Image.fromarray(a)
    if kind == "P":
        a = np.full((h, w, 3), 255, np.uint8)
        for k in range(12):
            x0 = w // 14 * (k + 1)
            top = int(h * (0.2 + 0.6 * rng.random()))
            a[top:h - h // 10, x0:x0 + max(w // 20, 1)] = rng.integers(0, 256, 3)
        a[h - h // 10, :] = 0
        return Image.fromarray(a).convert("P", palette=Image.Palette.ADAPTIVE, colors=64)
    base = np.stack([128 + 100 * np.sin(xx / 37 + c) * np.cos(yy / 53 - c) for c in range(3)], 2)
    return Image.fromarray(np.clip(base + rng.normal(0, 6, (h, w, 3)), 0, 255).astype(np.uint8))


def workload(kind):
    g = torch.Generator().manual_seed(0)                       # bench.py's configs[3] sizes
    hs = torch.randint(224, 1345, (32,), generator=g).tolist()
    ws = torch.randint(224, 1345, (32,), generator=g).tolist()
    rng = np.random.default_rng(1234)
    files = []
    for h, w in zip(hs, ws):
        b = io.BytesIO()
        content(kind, h, w, rng).save(b, "PNG")
        files.append(b.getvalue())
    return hs, ws, files


def run_kind(kind, dev, pool, reps, profile_calls, trace_dir):
    from tokenpacker_b200 import decode_png_batch, hd_preprocess_batch
    hs, ws, files = workload(kind)
    pinned = [torch.empty((h, w, 3), dtype=torch.uint8).pin_memory() for h, w in zip(hs, ws)]

    def pil_into(i):
        pinned[i].numpy()[...] = np.asarray(Image.open(io.BytesIO(files[i])).convert("RGB"))

    def path_a():
        list(pool.map(pil_into, range(len(files))))
        imgs = [p.to(dev, non_blocking=True) for p in pinned]
        out, _, _ = hd_preprocess_batch(imgs, 9, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        return out

    def path_b():
        out, _, _ = hd_preprocess_batch(decode_png_batch(files, dev), 9, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        return out

    def path_b0():
        decode_png_batch(files, dev, return_status=True)
        torch.cuda.synchronize()

    a, b = path_a(), path_b()                                   # warm-up, and the bit check
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{kind}: A and B differ"
    n_crops = a.shape[0]
    del a, b
    e2e = {"A_pil_pool16": [], "B_gpu_decode": [], "B0_gpu_decode_only": []}
    for _ in range(reps):
        for k, fn in (("A_pil_pool16", path_a), ("B_gpu_decode", path_b), ("B0_gpu_decode_only", path_b0)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            e2e[k].append((time.perf_counter() - t0) * 1e3)
    t0 = time.perf_counter()
    for f in files:
        Image.open(io.BytesIO(f)).convert("RGB")
    pil_one_core_ms = (time.perf_counter() - t0) * 1e3
    _, status = decode_png_batch(files, dev, return_status=True)
    st = status.cpu().numpy()
    assert (st[:, 0] == 0).all()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(profile_calls):
            decode_png_batch(files, dev, return_status=True)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if "png" in e.key:
            name = e.key.split("(")[0].split("::")[-1]
            kern[name] = {"calls": e.count, "avg_us_per_launch": e.device_time_total / max(e.count, 1),
                          "us_per_batch": e.device_time_total / profile_calls}
    if trace_dir:
        os.makedirs(trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(trace_dir, f"png_decode_{kind}.pt.trace.json"))
    return {"what": f"32 PNG files ({kind}, configs[3] sizes 224..1344, Pillow defaults) -> patch_num 9 -> {n_crops} bf16 crops",
            "png_bytes": sum(len(f) for f in files), "decoded_bytes": sum(h * w * 3 for h, w in zip(hs, ws)),
            "e2e_ms_median": {k: statistics.median(v) for k, v in e2e.items()}, "e2e_ms_min": {k: min(v) for k, v in e2e.items()},
            "e2e_bits_equal": True, "pil_one_core_ms_batch": pil_one_core_ms, "kernel_us": kern,
            "blocks": st[:, 1].tolist(), "chain_fallbacks": st[:, 2].tolist(), "candidates": st[:, 3].tolist()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--e2e-reps", type=int, default=5)
    ap.add_argument("--profile-calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-dir", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_png_decode: needs a CUDA device (there is no CPU measurement)")
    dev = torch.device("cuda", torch.cuda.current_device())
    pool = ThreadPoolExecutor(16)
    rec = {"card": card(dev), "host_threads_pool": 16, "cpu_count": os.cpu_count(),
           "kinds": {k: run_kind(k, dev, pool, args.e2e_reps, args.profile_calls, args.trace_dir) for k in ("L", "P", "RGB")}}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
