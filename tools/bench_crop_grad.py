"""Gradients to the pixels: the pixel-gradient step of CLIPVisionTowerB200 (``input_grad``) against transformers' bf16 CLIPVisionModel
with ``pixel_values.requires_grad_()`` and against our own 23-layer step without crop gradients; and the HD tiling backward
(tp_hd_tile_batch_backward) against F.interpolate's autograd.

    python tools/bench_crop_grad.py [--crops 64 231] [--rounds 3] [--out result.json]

Arms of the tower section, every one a forward of hidden states 12 / 16 / 22 / 23 and the backward of sum_j <d_j, hidden_states[j]>
(seeded bf16 d_j), all parameters frozen:
  pixel   CLIPVisionTowerB200 with input_grad: crops [N, 3, 336, 336] fp32 that require grad
  tower   CLIPVisionTowerB200(trainable_layers=23, train_embeddings=True) with only pre_layrnorm's two vectors requiring grad: the same
          23-layer and embedding-stage backward without the crop gradient, so pixel - tower is what the crop gradient costs
  hf      transformers' CLIPVisionModel, bf16, SDPA attention, eager autograd, pixel_values (bf16) requiring grad (skipped, and the JSON
          says so, when transformers is not importable)
with gradient checkpointing off and on at 64 crops, and on only at 231 crops (without it the saved sets of 231 crops do not fit in
80 GB for any arm).  Our arms follow the wrapped model's switch; transformers' is gradient_checkpointing_enable() in training mode.
Alternated rounds, CUDA events, medians with min-max; peak memory = max_memory_allocated during one step minus what was allocated
before it (weights and inputs excluded).

HD section: the 231-crop batch of bench.py's HD config (32 seeded sizes, patch_num 9).  Ours: the kernel alone (plan and tables staged
once), and the whole backward call (host plan, table upload, kernel).  Reference: oracle/crop_grad_oracle.tile in fp32 on the GPU
(F.interpolate, pad, split, thumbnail) and torch.autograd.grad of its crops.  Bytes: every d_crops element read once and every image
gradient written once, the least any adjoint moves.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_tower_oracle as cto  # noqa: E402
from oracle import crop_grad_oracle as cgo  # noqa: E402

HBM_GBS = 3350.0


def card(idx):
    """Name and power limit of the card, read (never set) in the same run as the measurement."""
    rec = {"name": torch.cuda.get_device_name(idx)}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = (v.strip() for v in q.stdout.strip().split(","))
        rec["power_limit_w"], rec["max_sm_mhz"] = float(pl), float(mx)
    except Exception as e:
        rec["power_limit_w"] = None
        rec["power_limit_error"] = repr(e)[:200]
    return rec


def timed(fn, reps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def peak_mib(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def stats(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--crops", type=int, nargs="+", default=[64, 231])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hd-reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_crop_grad: needs a CUDA device (there is no CPU measurement)")
    from tokenpacker_b200 import CLIPVisionTowerB200, hd
    from tokenpacker_b200._lib import check, lib
    dev = "cuda:0"
    result = {"card": card(0), "torch": torch.__version__}
    w = cto.round_bf16(cto.make_weights(23, seed=11, device=dev))
    frozen = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(dev).requires_grad_(False)
    pixel = CLIPVisionTowerB200(frozen)
    pixel.input_grad = True
    trained = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(dev)
    for name, p in trained.named_parameters():
        p.requires_grad_("pre_layrnorm" in name)
    tower = CLIPVisionTowerB200(trained, trainable_layers=23, train_embeddings=True)
    try:
        import transformers
        cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=24,
                                            patch_size=14, image_size=336, hidden_act="quick_gelu", layer_norm_eps=1e-5)
        cfg._attn_implementation = "sdpa"
        hf = transformers.CLIPVisionModel(cfg).to(dev, torch.bfloat16).requires_grad_(False)
        result["hf"] = f"transformers {transformers.__version__} CLIPVisionModel bf16, attention {hf.config._attn_implementation}"
    except Exception as e:              # measured arms stand without it; say why it is missing
        hf = None
        result["hf"] = f"not run: {repr(e)[:200]}"

    def hf_ckpt(on):
        if hf is None:
            return
        if on:
            hf.gradient_checkpointing_enable()
            hf.train()
        else:
            hf.gradient_checkpointing_disable()
            hf.eval()

    result["tower"] = []
    for n in args.crops:
        g = torch.Generator(device=dev).manual_seed(n)
        crops = cto.make_images(n, seed=n, device=dev).bfloat16().float()
        d = [(torch.randn(n, 577, 1024, generator=g, device=dev) * 0.1).bfloat16() for _ in range(4)]

        def step_pixel():
            x = crops.detach().requires_grad_(True)
            torch.autograd.backward(list(pixel.hidden_states(x)), d)

        def step_tower():
            torch.autograd.backward(list(tower.hidden_states(crops)), d)

        def step_hf():
            x = crops.detach().bfloat16().requires_grad_(True)
            hs = hf(pixel_values=x, output_hidden_states=True).hidden_states
            torch.autograd.backward([hs[j] for j in cto.OUT_LAYERS], d)

        arms = {"pixel": step_pixel, "tower": step_tower}
        if hf is not None:
            arms["hf"] = step_hf
        for ckpt in ([False, True] if n <= 64 else [True]):
            frozen.gradient_checkpointing = trained.gradient_checkpointing = ckpt
            hf_ckpt(ckpt)
            rec = {"crops": n, "checkpointing": ckpt, "ms": {}, "peak_mib": {}}
            times = {a: [] for a in arms}
            for a, fn in arms.items():
                fn()                                                        # warm-up: module loads, library algorithm choices
                rec["peak_mib"][a] = round(peak_mib(fn), 1)
            reps = 3 if n <= 64 else 1
            for _ in range(args.rounds):
                for a, fn in arms.items():
                    times[a].append(timed(fn, reps))
            rec["ms"] = {a: stats(v) for a, v in times.items()}
            rec["crop_grad_ms"] = rec["ms"]["pixel"]["median"] - rec["ms"]["tower"]["median"]
            if "hf" in arms:
                rec["speedup_vs_hf"] = rec["ms"]["hf"]["median"] / rec["ms"]["pixel"]["median"]
            print(json.dumps(rec), flush=True)
            result["tower"].append(rec)
            torch.cuda.empty_cache()

    # ---- HD tiling backward
    gs = torch.Generator().manual_seed(0)                                   # bench.py's HD config sizes
    hs = torch.randint(224, 1345, (32,), generator=gs).tolist()
    ws = torch.randint(224, 1345, (32,), generator=gs).tolist()
    gi = torch.Generator(device=dev).manual_seed(5)
    images = [torch.randn(3, h, wd, generator=gi, device=dev).requires_grad_(True) for h, wd in zip(hs, ws)]
    crops, hb, wb = hd.hd_tile_batch(images)
    n_crops = crops.shape[0]
    d_crops = torch.randn(crops.shape, generator=gi, device=dev)
    grads = torch.autograd.grad(crops, images, d_crops)
    sizes = list(zip(hs, ws))

    def ours_call():
        hd._tile_batch_backward(sizes, 9, d_crops)

    # the kernel alone: the tables of one call, staged once
    import ctypes as C
    from tokenpacker_b200 import _lib
    b = len(sizes)
    desc = (_lib.TpHdImage * b)()
    hb_c, wb_c, nc = (C.c_int * b)(), (C.c_int * b)(), C.c_int64(0)
    check(lib.tp_hd_tile_batch_plan((C.c_int64 * b)(*hs), (C.c_int64 * b)(*ws), None, b, 9, desc, None, hb_c, wb_c, C.byref(nc)), "plan")
    outs = [torch.empty(3, h, wd, device=dev) for h, wd in sizes]
    ptrs = (C.c_void_p * b)(*[o.data_ptr() for o in outs])
    words, most = C.c_int64(0), C.c_int64(0)
    check(lib.tp_hd_tile_batch_backward_plan(desc, b, ptrs, None, None, C.byref(words), C.byref(most)), "bwd plan")
    gdesc = (_lib.TpHdImageGrad * b)()
    taps = torch.empty(words.value, dtype=torch.int32)
    check(lib.tp_hd_tile_batch_backward_plan(desc, b, ptrs, gdesc, C.cast(taps.data_ptr(), C.POINTER(C.c_int32)), C.byref(words),
                                             C.byref(most)), "bwd plan")
    d_desc = torch.frombuffer(bytearray(bytes(desc)), dtype=torch.uint8).to(dev)
    d_g = torch.frombuffer(bytearray(bytes(gdesc)), dtype=torch.uint8).to(dev)
    d_taps = taps.to(dev)
    stream = torch.cuda.current_stream().cuda_stream

    def ours_kernel():
        check(lib.tp_hd_tile_batch_backward(d_desc.data_ptr(), d_g.data_ptr(), d_taps.data_ptr(), b, most.value, d_crops.data_ptr(), stream),
              "bwd")

    ours_kernel()
    torch.cuda.synchronize()
    exact = all(torch.equal(o, gr) for o, gr in zip(outs, grads))
    leaves = [im.detach().clone().requires_grad_(True) for im in images]
    ref_crops = torch.cat([cgo.tile(x, 9)[0] for x in leaves], dim=0)

    def ref_backward():
        torch.autograd.grad(ref_crops, leaves, d_crops, retain_graph=True)

    ref_grads = torch.autograd.grad(ref_crops, leaves, d_crops, retain_graph=True)
    rel = max(float((a.double() - r.double()).norm() / r.double().norm()) for a, r in zip(grads, ref_grads))
    fns = {"ours_kernel": ours_kernel, "ours_call": ours_call, "interpolate_autograd": ref_backward}
    t = {k: [] for k in fns}
    for fn in fns.values():
        for _ in range(3):
            fn()
    for _ in range(args.rounds):
        for k, fn in fns.items():
            t[k].append(timed(fn, args.hd_reps))
    nbytes = (d_crops.numel() + sum(3 * h * wd for h, wd in sizes)) * 4
    kern = statistics.median(t["ours_kernel"])
    result["hd_backward"] = {"images": b, "crops": n_crops, "ms": {k: stats(v) for k, v in t.items()},
                             "kernel_bytes_min": nbytes, "kernel_gbs": nbytes / kern / 1e6,
                             "kernel_share_of_hbm_peak": nbytes / kern / 1e6 / HBM_GBS,
                             "kernel_equals_autograd_path": exact, "rel_rms_vs_interpolate_autograd_fp32": rel}
    print(json.dumps(result["hd_backward"]), flush=True)
    line = json.dumps(result)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
