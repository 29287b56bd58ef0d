"""CLIP-ViT-L/14-336 tower: transformers' bf16 CLIPVisionModel (arm A) against CLIPVisionTowerB200.hidden_states (arm B).

    python tools/bench_clip_tower.py [--crops 64 231] [--rounds 5] [--out result.json] [--dtype float16]

Seeded weights at the real shapes (oracle/clip_tower_oracle.py).  Arm A is transformers' CLIPVisionModel built from config, bf16,
SDPA attention, called as the released recipe calls it (output_hidden_states=True, then hidden states 12 / 16 / 22 / 23 picked); when
transformers is not importable the oracle's bf16 eager restatement (same rounding points, F.scaled_dot_product_attention) stands in,
and the JSON says which ran.  Alternated rounds, CUDA events, medians.  Work per crop is algorithmic (formula below), not measured.
Errors: each arm's hidden states against the fp64 oracle on the first crops of the batch (rel-RMS over the four states).

--dtype float16 measures the evaluation / serving precision instead: arm A is transformers' CLIPVisionModel in fp16 (the oracle's fp16
eager restatement without transformers), arm B CLIPVisionTowerB200(dtype=torch.float16), and arm C — alternated in the same rounds —
our bf16 tower (dtype=None) on the same weights cast to bf16.  The weights are rounded to fp16 first, so the fp16 arms compute from
exactly the fp64 oracle's weights; the crops are bf16, as the preprocessing produces them.  No whole-path section in this mode.
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

from oracle import clip_tower_f16_oracle as ct16  # noqa: E402
from oracle import clip_tower_oracle as cto  # noqa: E402


def tower_gflop_per_crop(layers=23, t=577, d=1024, f=4096, patches=576, k=588):
    """2 FLOP per multiply-add: per layer q/k/v/out (4 d^2) and fc1/fc2 (2 d f) linears, plus S = QK^T and PV (2 t^2 d); and the patch
    embedding (patches x k x d).  = 366.03 GF for the 23 layers hidden_states[23] needs (arm A runs 24 layers: 381.9 GF of
    work; both arms are rated on the 366.03 GF the result needs)."""
    linears = 2 * t * (4 * d * d + 2 * d * f)
    attention = 2 * 2 * t * t * d
    return (layers * (linears + attention) + 2 * patches * k * d) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--crops", type=int, nargs="+", default=[64, 231])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--err-crops", type=int, default=4)
    ap.add_argument("--path-crops", type=int, default=64)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dtype", choices=["bfloat16", "float16"], default="bfloat16")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    dev = "cuda:0"
    from tokenpacker_b200 import CLIPVisionTowerB200
    f16 = args.dtype == "float16"
    dt = torch.float16 if f16 else torch.bfloat16
    if f16:
        w = {k: v.half().float() for k, v in cto.make_weights(23, seed=11, device=dev).items()}
    else:
        w = cto.round_bf16(cto.make_weights(23, seed=11, device=dev))
    wb = {k: v.to(dt) for k, v in w.items()}
    ours = CLIPVisionTowerB200(cto.FakeCLIPVisionModel(wb), dtype=dt if f16 else None)
    try:
        import transformers
        cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=24,
                                            image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
        hf = transformers.CLIPVisionModel(cfg).to(dev, dt).eval()
        sd = hf.state_dict()
        sd.update({"vision_model." + k: v for k, v in wb.items()})
        hf.load_state_dict(sd)
        arm_a = (f"transformers {transformers.__version__} CLIPVisionModel {args.dtype}, attention {hf.config._attn_implementation} "
                 "(24 layers + post_layernorm run)")

        def run_a(x):
            hs = hf(pixel_values=x.to(dt), output_hidden_states=True).hidden_states     # clip_encoder.py:59: images to the tower's dtype
            return tuple(hs[i] for i in cto.OUT_LAYERS)
    except ImportError:
        arm_a = f"oracle {args.dtype} eager restatement (transformers not importable)"

        def run_a(x):
            hs = ct16.forward_eager(w, x, 23, dt) if f16 else cto.forward_bf16_eager(w, x, 23)
            return tuple(hs[i] for i in cto.OUT_LAYERS)

    def run_b(x):
        return ours.hidden_states(x)

    arms = (("A", run_a), ("B", run_b))
    if f16:
        ours_bf16 = CLIPVisionTowerB200(cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}))

        def run_c(x):
            return ours_bf16.hidden_states(x)

        arms += (("C", run_c),)

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    gf = tower_gflop_per_crop()
    result = {"bench": "clip_tower", "gpu": smi, "arm_a": arm_a, "arm_b": "CLIPVisionTowerB200.hidden_states", "gflop_per_crop": round(gf, 2),
              "workloads": []}
    if f16:
        result.update(bench="clip_tower_f16", arm_b="CLIPVisionTowerB200(dtype=torch.float16).hidden_states (fp16 outputs)",
                      arm_c="CLIPVisionTowerB200(dtype=None).hidden_states on the same weights cast to bf16 (bf16 outputs)")
    with torch.no_grad():
        for n in args.crops:
            x = cto.make_images(n, seed=n, device=dev).bfloat16()
            times = {name: [] for name, _ in arms}
            mem = {}
            for name, fn in arms:                                   # warm-up, peak memory of one call on its own
                fn(x)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                out = fn(x)
                torch.cuda.synchronize()
                mem[name] = torch.cuda.max_memory_allocated() - base
                del out
            for _ in range(args.rounds):
                for name, fn in arms:
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    out = fn(x)
                    e.record()
                    torch.cuda.synchronize()
                    times[name].append(s.elapsed_time(e))
                    del out
            k = min(args.err_crops, n)
            ref = cto.forward(w, x[:k].double(), 23, torch.float64)
            errs = {}
            for name, fn in arms:
                got = fn(x[:k])
                errs[name] = [float((g.double() - ref[i]).norm() / ref[i].norm()) for g, i in zip(got, cto.OUT_LAYERS)]
            del ref
            row = {"crops": n}
            for name, _ in arms:
                ms = statistics.median(times[name])
                row[name] = {"ms_median": round(ms, 3), "ms_all": [round(t, 3) for t in times[name]],
                             "tflops_algorithmic": round(gf * n / ms, 1), "peak_bytes_above_inputs": int(mem[name]),
                             "rel_rms_vs_fp64_hs12_16_22_23": [float(f"{v:.3e}") for v in errs[name]]}
            row["speedup_B_over_A"] = round(row["A"]["ms_median"] / row["B"]["ms_median"], 3)
            if f16:
                row["time_B_over_C"] = round(row["B"]["ms_median"] / row["C"]["ms_median"], 3)
            result["workloads"].append(row)
            torch.cuda.empty_cache()
        if f16:
            line = json.dumps(result)
            print(line)
            if args.out:
                with open(args.out, "w") as f:
                    f.write(line + "\n")
            return
        # whole path: (A) transformers' tower, feature_select's [:,1:] + torch.cat, TokenPackerB200.forward against (B) our tower and
        # forward_hidden_states (the four layers read in place); the 144-token s = 2 projector at hidden 4096
        from tokenpacker_b200 import TokenPackerB200
        torch.manual_seed(0)
        proj = TokenPackerB200(hidden_size=4096, scale_factor=2).to(dev, torch.bfloat16).eval()

        def path_a(x):
            hs = run_a(x)
            return proj((hs[3][:, 1:], torch.cat([h[:, 1:] for h in hs], dim=-1)))

        def path_b(x):
            return proj.forward_hidden_states(list(run_b(x)))

        x = cto.make_images(args.path_crops, seed=3, device=dev).bfloat16()
        times = {"A": [], "B": []}
        for fn in (path_a, path_b):
            fn(x)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for name, fn in (("A", path_a), ("B", path_b)):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                out = fn(x)
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e))
                del out
        result["whole_path"] = {"crops": args.path_crops, "what": "tower + projector (hidden 4096, s = 2): A = transformers tower + cat + "
                                "forward, B = CLIPVisionTowerB200 + forward_hidden_states",
                                "A_ms_median": round(statistics.median(times["A"]), 3), "B_ms_median": round(statistics.median(times["B"]), 3),
                                "A_ms_all": [round(t, 3) for t in times["A"]], "B_ms_all": [round(t, 3) for t in times["B"]]}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
