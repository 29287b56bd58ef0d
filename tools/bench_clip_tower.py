"""CLIP-ViT-L/14-336 tower: transformers' bf16 CLIPVisionModel (arm A) against CLIPVisionTowerB200.hidden_states (arm B).

    python tools/bench_clip_tower.py [--crops 64 231] [--rounds 5] [--out result.json]

Seeded weights at the real shapes (oracle/clip_tower_oracle.py).  Arm A is transformers' CLIPVisionModel built from config, bf16,
SDPA attention, called as the released recipe calls it (output_hidden_states=True, then hidden states 12 / 16 / 22 / 23 picked); when
transformers is not importable the oracle's bf16 eager restatement (same rounding points, F.scaled_dot_product_attention) stands in,
and the JSON says which ran.  Alternated rounds, CUDA events, medians.  Work per crop is algorithmic (formula below), not measured.
Errors: each arm's hidden states against the fp64 oracle on the first crops of the batch (rel-RMS over the four states).
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
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    dev = "cuda:0"
    from tokenpacker_b200 import CLIPVisionTowerB200
    w = cto.round_bf16(cto.make_weights(23, seed=11, device=dev))
    wb = {k: v.bfloat16() for k, v in w.items()}
    ours = CLIPVisionTowerB200(cto.FakeCLIPVisionModel(wb))
    try:
        import transformers
        cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=24,
                                            image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
        hf = transformers.CLIPVisionModel(cfg).to(dev, torch.bfloat16).eval()
        sd = hf.state_dict()
        sd.update({"vision_model." + k: v for k, v in wb.items()})
        hf.load_state_dict(sd)
        arm_a = (f"transformers {transformers.__version__} CLIPVisionModel bf16, attention {hf.config._attn_implementation} "
                 "(24 layers + post_layernorm run)")

        def run_a(x):
            hs = hf(pixel_values=x, output_hidden_states=True).hidden_states
            return tuple(hs[i] for i in cto.OUT_LAYERS)
    except ImportError:
        arm_a = "oracle bf16 eager restatement (transformers not importable)"

        def run_a(x):
            hs = cto.forward_bf16_eager(w, x, 23)
            return tuple(hs[i] for i in cto.OUT_LAYERS)

    def run_b(x):
        return ours.hidden_states(x)

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    gf = tower_gflop_per_crop()
    result = {"bench": "clip_tower", "gpu": smi, "arm_a": arm_a, "arm_b": "CLIPVisionTowerB200.hidden_states", "gflop_per_crop": round(gf, 2),
              "workloads": []}
    with torch.no_grad():
        for n in args.crops:
            x = cto.make_images(n, seed=n, device=dev).bfloat16()
            times = {"A": [], "B": []}
            mem = {}
            for name, fn in (("A", run_a), ("B", run_b)):          # warm-up, peak memory of one call on its own
                fn(x)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                out = fn(x)
                torch.cuda.synchronize()
                mem[name] = torch.cuda.max_memory_allocated() - base
                del out
            for _ in range(args.rounds):
                for name, fn in (("A", run_a), ("B", run_b)):
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
            for name, fn in (("A", run_a), ("B", run_b)):
                got = fn(x[:k])
                errs[name] = [float((g.double() - ref[i]).norm() / ref[i].norm()) for g, i in zip(got, cto.OUT_LAYERS)]
            del ref
            row = {"crops": n}
            for name in ("A", "B"):
                ms = statistics.median(times[name])
                row[name] = {"ms_median": round(ms, 3), "ms_all": [round(t, 3) for t in times[name]],
                             "tflops_algorithmic": round(gf * n / ms, 1), "peak_bytes_above_inputs": int(mem[name]),
                             "rel_rms_vs_fp64_hs12_16_22_23": [float(f"{v:.3e}") for v in errs[name]]}
            row["speedup_B_over_A"] = round(row["A"]["ms_median"] / row["B"]["ms_median"], 3)
            result["workloads"].append(row)
            torch.cuda.empty_cache()
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
