"""Non-HD CLIP input on the GPU against the host processor: kernel times per pass and end-to-end times from pinned host buffers.

    python tools/bench_clip_preprocess.py [--reps 50] [--e2e-reps 5] [--out result.json]

Workload: BASELINE configs[3]'s 32 image sizes (seeded as in bench.py, 224..1344) with seeded uint8 pixels, in pad mode (finetuning and
eval: expand2square, then the processor) and square mode (pretraining: the processor alone).  Prints one JSON line (and writes it to
--out).

  kernels alone (the plan tables resident on the device): tp_clip_preprocess_batch -> bf16 [32, 3, 336, 336]; CUDA events over --reps
    calls, best of 3 rounds, and each pass's own device time from torch.profiler
    algorithmic bytes = every source byte read once + the workspace written and read once + the output written once
  end to end from pinned host uint8 images [h, w, 3], each path ending in a device synchronise (host clock), A and B alternated
    (A)  what the reference runs: expand2square (pad) + the slow CLIP processor (transformers' CLIPImageProcessorPil, the
         openai/clip-vit-large-patch14-336 configuration) per image over a thread pool as wide as the host's cores, np.stack,
         pinned float32, upload, .to(bfloat16)
    (B)  upload uint8, clip_preprocess_batch(dtype=torch.bfloat16)
  A and B are asserted to give equal bits.  Arm A needs Pillow and transformers; without them B is recorded alone and the record
  says why.  Writes nothing but --out.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_hd_preprocess import HBM_GBS, card, event_ms   # noqa: E402


def host_processor():
    """(expand2square, processor) of the host path, or the reason it is unavailable."""
    try:
        from PIL import Image
        from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
        from oracle.gen_golden_clip_preprocess import PROCESSOR
    except Exception as e:                       # noqa: BLE001  (a missing optional dependency: arm A is skipped and says why)
        return None, repr(e)[:200]
    from oracle.clip_preprocess_oracle import BACKGROUND
    proc = CLIPImageProcessorPil(**PROCESSOR)

    def expand2square(pil):                      # mm_utils.py:14-25 with Image.new + paste
        w, h = pil.size
        if w == h:
            return pil
        out = Image.new(pil.mode, (max(w, h), max(w, h)), BACKGROUND)
        out.paste(pil, (0, (w - h) // 2) if w > h else ((h - w) // 2, 0))
        return out

    def one(px, mode):
        pil = Image.fromarray(px)
        if mode == "pad":
            pil = expand2square(pil)
        return proc.preprocess(pil, return_tensors="np")["pixel_values"][0]
    return one, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--e2e-reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip_preprocess: needs a CUDA device (there is no CPU measurement)")
    from tokenpacker_b200 import clip_preprocess_batch
    from tokenpacker_b200._lib import check, lib
    import ctypes as C
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = torch.cuda.current_stream(dev).cuda_stream

    g = torch.Generator().manual_seed(0)                       # bench.py's configs[3] sizes
    hs = torch.randint(224, 1345, (32,), generator=g).tolist()
    ws = torch.randint(224, 1345, (32,), generator=g).tolist()
    rng = np.random.default_rng(1234)
    host_np = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in zip(hs, ws)]
    host_u8 = [torch.from_numpy(p).pin_memory() for p in host_np]
    dev_u8 = [u.to(dev) for u in host_u8]
    src_bytes = sum(h * w * 3 for h, w in zip(hs, ws))
    out_bytes = 32 * 3 * 336 * 336 * 2
    rec = {"what": "32 images (configs[3] sizes 224..1344) -> [32, 3, 336, 336] bf16", "card": card(dev), "source_bytes": src_bytes,
           "kernel": {}, "e2e": {}}

    one, why = host_processor()
    pool = ThreadPoolExecutor(max_workers=os.cpu_count() or 1)
    if one is None:
        rec["arm_A"] = "not run: " + why

    for mode in ("pad", "square"):
        # ------------------------------------------------------------ kernels alone
        ref, (t, soff, coff, plan, wsb, table) = clip_preprocess_batch(dev_u8, mode, dtype=torch.bfloat16, _return_launch=True)
        torch.cuda.synchronize()
        tabs = t.clone()                                       # the staging buffer is shared by later calls: keep a copy
        out = torch.empty_like(ref)

        def run(tabs=tabs, soff=soff, coff=coff, plan=plan, wsb=wsb, table=table, out=out):
            check(lib.tp_clip_preprocess_batch(C.addressof(plan), tabs.data_ptr(), tabs.data_ptr() + soff, tabs.data_ptr() + coff, 32,
                                               table.data_ptr(), 1, out.data_ptr(), wsb.data_ptr(), wsb.numel(), stream),
                  "tp_clip_preprocess_batch")
        rounds = [event_ms(run, args.reps) for _ in range(3)]
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
        ws_bytes = int(wsb.numel())
        by = src_bytes + 2 * ws_bytes + out_bytes
        ms = min(rounds)
        passes = {}
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                run()
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            name = ev.key
            if "clip_resample_h_kernel" in name or "clip_resample_v_kernel" in name:
                key = "horizontal" if "_h_" in name else "vertical"
                dt = getattr(ev, "device_time_total", None)
                if dt is None:
                    dt = ev.cuda_time_total
                passes[key] = {"ms": dt / 1e3 / max(ev.count, 1), "launches": ev.count}
        rec["kernel"][mode] = {"ms": ms, "ms_rounds": rounds, "passes_profiler": passes, "workspace_bytes": ws_bytes,
                               "algorithmic_bytes": by, "gbs": by / (ms * 1e-3) / 1e9, "frac_of_3350_gbs": by / (ms * 1e-3) / 1e9 / HBM_GBS}
        del run, out, tabs

        # ------------------------------------------------------------ end to end from pinned host buffers
        host_f32 = torch.empty((32, 3, 336, 336), dtype=torch.float32).pin_memory()

        def path_a(mode=mode, host_f32=host_f32):
            outs = list(pool.map(lambda px: one(px, mode), host_np))
            host_f32.copy_(torch.from_numpy(np.stack(outs)))
            o = host_f32.to(dev, non_blocking=True).to(torch.bfloat16)
            torch.cuda.synchronize()
            return o

        def path_b(mode=mode):
            imgs = [u.to(dev, non_blocking=True) for u in host_u8]
            o = clip_preprocess_batch(imgs, mode, dtype=torch.bfloat16)
            torch.cuda.synchronize()
            return o

        paths = {"B_u8_gpu": path_b}
        if one is not None:
            paths = {"A_host_processor": path_a, "B_u8_gpu": path_b}
        b = path_b()
        assert torch.equal(b.view(torch.int16), ref.view(torch.int16))
        if one is not None:
            a = path_a()                                           # warm-up, and the bit check
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"A and B differ ({mode})"
        times = {k: [] for k in paths}
        for _ in range(args.e2e_reps):
            for k, fn in paths.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                times[k].append((time.perf_counter() - t0) * 1e3)
        rec["e2e"][mode] = {"ms_median": {k: statistics.median(v) for k, v in times.items()}, "ms_min": {k: min(v) for k, v in times.items()},
                            "bits_equal": one is not None, "upload_bytes": {"A": out_bytes * 2, "B": src_bytes}}
    rec["host_threads"] = os.cpu_count()
    pool.shutdown()
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
