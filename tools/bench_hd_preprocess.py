"""Decoded 8-bit HD input on the GPU against normalising on the host: kernel times and end-to-end times from pinned host buffers.

    python tools/bench_hd_preprocess.py [--reps 50] [--e2e-reps 10] [--out result.json]

Workload: BASELINE configs[3]'s HD batch (32 images, sizes seeded as in bench.py, patch_num 9, 231 crops) with seeded uint8 pixels.
Prints one JSON line (and writes it to --out).

  kernel alone (CUDA events over --reps launches after warm-up, plan tables resident on the device)
    (i)   tp_hd_tile_batch            float32 [3,h,w] normalised source -> float32 crops
    (ii)  tp_hd_preprocess_batch      uint8 [h,w,3] source               -> float32 crops
    (iii) tp_hd_preprocess_batch      uint8 [h,w,3] source               -> bf16 crops
    algorithmic bytes = every source byte read once + every crop byte written once; GB/s against 3.35 TB/s (H100 SXM HBM3)
  end to end from pinned host uint8 images [h,w,3], each path ending in a device synchronise (host clock), A and B alternated
    (A)  ToTensor + Normalize on the host (the torch CPU ops torchvision runs) into pinned float32, upload, hd_tile_batch, .to(bf16)
    (A') as A, from images already normalised into pinned float32 (the upload + kernel + cast part of A alone)
    (B)  upload uint8, hd_preprocess_batch(dtype=torch.bfloat16)
  A and B are asserted to give equal bits.  Writes nothing but --out.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_GBS = 3350.0


def card(dev):
    """Name and power limit of the card, read (never set) in the same run as the measurement."""
    idx = dev.index or 0
    rec = {"name": torch.cuda.get_device_name(idx)}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = (v.strip() for v in q.stdout.strip().split(","))
        rec["power_limit_w"], rec["max_sm_mhz"] = float(pl), float(mx)
    except Exception as e:              # the measurement stands without it; say why it is missing
        rec["power_limit_w"] = None
        rec["power_limit_error"] = repr(e)[:200]
    return rec


def event_ms(fn, reps, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--e2e-reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hd_preprocess: needs a CUDA device (there is no CPU measurement)")
    from tokenpacker_b200 import hd_preprocess_batch, hd_tile_batch
    from tokenpacker_b200._lib import check, lib
    from tokenpacker_b200.hd import CLIP_MEAN, CLIP_STD, norm_table
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = torch.cuda.current_stream(dev).cuda_stream

    g = torch.Generator().manual_seed(0)                       # bench.py's configs[3] sizes
    hs = torch.randint(224, 1345, (32,), generator=g).tolist()
    ws = torch.randint(224, 1345, (32,), generator=g).tolist()
    rng = np.random.default_rng(1234)
    host_u8 = [torch.from_numpy(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)).pin_memory() for h, w in zip(hs, ws)]
    mean = torch.tensor(CLIP_MEAN, dtype=torch.float32)[:, None, None]
    std = torch.tensor(CLIP_STD, dtype=torch.float32)[:, None, None]
    host_f32 = [torch.empty((3, h, w), dtype=torch.float32).pin_memory() for h, w in zip(hs, ws)]

    def normalise_on_host():
        for u, f in zip(host_u8, host_f32):           # ToTensor (permute, float, div 255) + Normalize (sub mean, div std)
            torch.div(u.permute(2, 0, 1).float().div(255).sub_(mean), std, out=f)

    normalise_on_host()
    table = norm_table()
    assert torch.equal(host_f32[0], torch.stack([table[c][host_u8[0][:, :, c].long()] for c in range(3)]))

    # ---------------------------------------------------------------- kernel alone
    dev_u8 = [u.to(dev) for u in host_u8]
    dev_f32 = [f.to(dev) for f in host_f32]
    crops32, hb, wb, (t, toff, n) = hd_tile_batch(dev_f32, 9, _return_launch=True)
    tab_i = t[:toff + n * 12].clone()                          # the staging buffer is shared by later calls: keep a copy
    ref32 = crops32.clone()
    kernels = {}

    def run_i():
        check(lib.tp_hd_tile_batch(tab_i.data_ptr(), tab_i.data_ptr() + toff, n, crops32.data_ptr(), stream), "tp_hd_tile_batch")
    kernels["i_f32_to_f32"] = (run_i, 4, 4)
    outs = {}
    for name, dt, code, ob in (("ii_u8_to_f32", torch.float32, 0, 4), ("iii_u8_to_bf16", torch.bfloat16, 1, 2)):
        c, _, _, (t2, soff, toff2, n2, ntab) = hd_preprocess_batch(dev_u8, 9, dtype=dt, _return_launch=True)
        tab = t2[:toff2 + n2 * 12].clone()
        outs[name] = c

        def run(tab=tab, soff=soff, toff2=toff2, n2=n2, ntab=ntab, c=c, code=code):
            check(lib.tp_hd_preprocess_batch(tab.data_ptr(), tab.data_ptr() + soff, tab.data_ptr() + toff2, n2, ntab.data_ptr(), code,
                                             c.data_ptr(), stream), "tp_hd_preprocess_batch")
        kernels[name] = (run, 1, ob)
    src_px = sum(h * w * 3 for h, w in zip(hs, ws))
    crop_el = n * 3 * 336 * 336
    rec = {"what": "32 images (configs[3] sizes 224..1344), patch_num 9 -> %d crops [3,336,336]" % n, "card": card(dev),
           "source_pixels": src_px, "crops": n, "kernel": {}}
    # interleave the three kernels over three rounds; report each one's best round (another user's work can share the card)
    times = {k: [] for k in kernels}
    for _ in range(3):
        for k, (fn, _, _) in kernels.items():
            times[k].append(event_ms(fn, args.reps))
    for k, (fn, sb, ob) in kernels.items():
        ms = min(times[k])
        by = src_px * sb + crop_el * ob
        rec["kernel"][k] = {"ms": ms, "ms_rounds": times[k], "algorithmic_bytes": by, "gbs": by / (ms * 1e-3) / 1e9,
                            "frac_of_3350_gbs": by / (ms * 1e-3) / 1e9 / HBM_GBS}
    torch.cuda.synchronize()
    assert torch.equal(crops32, ref32) and torch.equal(outs["ii_u8_to_f32"], ref32)
    assert torch.equal(outs["iii_u8_to_bf16"].view(torch.int16), ref32.to(torch.bfloat16).view(torch.int16))
    del kernels, outs, crops32, ref32, dev_u8, dev_f32

    # ---------------------------------------------------------------- end to end from pinned host buffers
    def path_a(normalise=True):
        if normalise:
            normalise_on_host()
        imgs = [f.to(dev, non_blocking=True) for f in host_f32]
        crops, _, _ = hd_tile_batch(imgs, 9)
        out = crops.to(torch.bfloat16)
        torch.cuda.synchronize()
        return out

    def path_b():
        imgs = [u.to(dev, non_blocking=True) for u in host_u8]
        out, _, _ = hd_preprocess_batch(imgs, 9, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        return out

    e2e = {"A_host_normalise": [], "A_prenormalised": [], "B_u8": []}
    a, b = path_a(), path_b()                                   # warm-up, and the bit check
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "A and B differ"
    del a, b
    for _ in range(args.e2e_reps):
        for k, fn in (("A_host_normalise", path_a), ("B_u8", path_b), ("A_prenormalised", lambda: path_a(False)), ("B_u8", path_b)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            e2e[k].append((time.perf_counter() - t0) * 1e3)
    rec["e2e_ms_median"] = {k: statistics.median(v) for k, v in e2e.items()}
    rec["e2e_ms_min"] = {k: min(v) for k, v in e2e.items()}
    rec["e2e_upload_bytes"] = {"A": src_px * 4, "B": src_px}
    rec["e2e_bits_equal"] = True
    rec["torch_threads"] = torch.get_num_threads()
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
