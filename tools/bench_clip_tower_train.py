"""Training step of the CLIP-ViT-L/14-336 tower with its last K layers trainable: forward + backward of
CLIPVisionTowerB200(trainable_layers=K).hidden_states (arm B) against the same step in eager PyTorch under autograd (arm A).

    python tools/bench_clip_tower_train.py [--crops 64] [--layers 2 4 12] [--rounds 5] [--out result.json]

Seeded weights at the real shapes (oracle/clip_tower_oracle.py).  Arm A: the oracle's bf16 eager restatement of transformers' tower
(same rounding points, F.scaled_dot_product_attention), layers 0 .. 22 - K under torch.no_grad(), layers 23 - K .. 22 under autograd
— what freezing the bottom of CLIPVisionModel gives.  If transformers is importable, arm C is its CLIPVisionModel in bf16 with the same
layers unfrozen (it runs all 24 layers and keeps every hidden state).  Arm D is arm B with gradient checkpointing (the wrapped model's
``gradient_checkpointing`` switch on: include/tokenpacker_b200_clip_tower_ckpt.h), arm E arm C after ``gradient_checkpointing_enable()``.
The loss is a fixed weighted sum of hidden states 12 / 16 / 22 / 23 (those that depend on a trainable layer), so the backward starts from
four dense gradients as the projector's input gradients do.  Alternated rounds, CUDA events around forward + backward, medians; peak
memory of one step above what was allocated before it.  Work per crop is algorithmic (formula below), not measured.

Before an arm runs, its peak is predicted from the size queries (``predict_bytes``) and compared with torch.cuda.mem_get_info(); an arm
the prediction rules out is recorded as "does not fit: needs X GB" instead of being run into an out-of-memory error.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_tower_oracle as cto  # noqa: E402


def step_gflop_per_crop(k, layers=23, t=577, d=1024, f=4096, patches=576, kk=588):
    """2 FLOP per multiply-add.  Forward: the 23 layers' linears (4 d^2 + 2 d f per token) and attention (2 t^2 d per product, two
    products), plus the patch embedding.  Backward of a trainable layer: a dgrad and a wgrad per linear (2x the forward's linears) and
    five attention products (S, dP, dV, dK, dQ: 2.5x the forward's two)."""
    linears = 2 * t * (4 * d * d + 2 * d * f)
    attention = 2 * 2 * t * t * d
    forward = layers * (linears + attention) + 2 * patches * kk * d
    backward = k * (2 * linears + 2.5 * attention)
    return forward / 1e9, backward / 1e9


# Arms without a size query of their own are predicted from ours in the same mode, times the ratio of their peak to ours observed at
# 64 crops (tools/bench_clip_tower_train_h100.json: eager <= 0.8 - 1.1x, transformers 1.2 - 1.35x); the margin covers allocator slack.
_PREDICT_SCALE = {"A": 1.1, "B": 1.0, "C": 1.35, "D": 1.0, "E": 1.35}
_MARGIN = 1.1


def predict_bytes(lib, arm, n, k):
    """Peak bytes of one step above its start: what is kept between forward and backward, plus the larger of the forward's workspace
    and the backward's workspace with the parameter gradients (16 tensors per layer, 12.6 M elements) and the four outputs' gradients."""
    outs = 4 * n * 577 * 1024 * 2
    grads = k * 12_596_224 * 2 + outs
    if arm in ("D", "E"):
        kept, fwd, bwd = (lib.tp_clip_tower_ckpt_saved_bytes(n, k), lib.tp_clip_tower_workspace_bytes(n),
                          lib.tp_clip_tower_ckpt_backward_workspace_bytes(n, k))
    else:
        kept, fwd, bwd = (lib.tp_clip_tower_train_saved_bytes(n, k), lib.tp_clip_tower_train_workspace_bytes(n, k),
                          lib.tp_clip_tower_backward_workspace_bytes(n, k))
    if arm in ("C", "E"):
        kept += 25 * n * 577 * 1024 * 2                                # transformers keeps every hidden state
    return int(_PREDICT_SCALE[arm] * (kept + outs + max(fwd, bwd + grads)))


def eager_layer(x, p):
    n = x.shape[0]
    y = F.layer_norm(x, (1024,), p["layer_norm1.weight"], p["layer_norm1.bias"], 1e-5)
    sh = lambda t: t.view(n, 577, 16, 64).transpose(1, 2)
    q, k, v = (sh(F.linear(y, p[f"self_attn.{a}_proj.weight"], p[f"self_attn.{a}_proj.bias"])) for a in "qkv")
    a = F.scaled_dot_product_attention(q, k, v, scale=0.125).transpose(1, 2).reshape(n, 577, 1024)
    x = x + F.linear(a, p["self_attn.out_proj.weight"], p["self_attn.out_proj.bias"])
    y = F.layer_norm(x, (1024,), p["layer_norm2.weight"], p["layer_norm2.bias"], 1e-5)
    return x + F.linear(cto.quick_gelu(F.linear(y, p["mlp.fc1.weight"], p["mlp.fc1.bias"])), p["mlp.fc2.weight"], p["mlp.fc2.bias"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--crops", type=int, default=64)
    ap.add_argument("--layers", type=int, nargs="+", default=[2, 4, 12])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    dev = "cuda:0"
    from tokenpacker_b200 import CLIPVisionTowerB200, _lib
    w = cto.make_weights(23, seed=11, device=dev)
    wb = {k: v.bfloat16() for k, v in w.items()}
    del w
    n = args.crops
    x = cto.make_images(n, seed=n, device=dev).bfloat16()
    g = torch.Generator(device=dev).manual_seed(5)
    d_outs = [(torch.randn(n, 577, 1024, generator=g, device=dev) * 0.1).bfloat16() for _ in cto.OUT_LAYERS]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    result = {"bench": "clip_tower_train", "gpu_name_powerlimit_maxsmclock_smclock": smi, "crops": n,
              "arm_a": "oracle bf16 eager restatement under autograd, frozen layers under no_grad",
              "arm_b": "CLIPVisionTowerB200(trainable_layers=K).hidden_states + backward",
              "arm_d": "arm B with the wrapped model's gradient_checkpointing switch on", "workloads": []}
    try:
        import transformers
        cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=24,
                                            image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
        hf = transformers.CLIPVisionModel(cfg).to(dev, torch.bfloat16)
        sd = hf.state_dict()
        sd.update({"vision_model." + k: v for k, v in wb.items()})
        hf.load_state_dict(sd)
        hf_ckpt = transformers.CLIPVisionModel(cfg).to(dev, torch.bfloat16).train()      # transformers recomputes only in training
        hf_ckpt.load_state_dict(sd)
        hf_ckpt.gradient_checkpointing_enable()
        del sd
        result["arm_c"] = f"transformers {transformers.__version__} CLIPVisionModel bf16 under autograd, same layers unfrozen"
        result["arm_e"] = "arm C after gradient_checkpointing_enable()"
    except ImportError:
        hf = None

    for k in args.layers:
        first = 23 - k
        used = [i for i, j in enumerate(cto.OUT_LAYERS) if j - 1 >= first]
        model = cto.FakeCLIPVisionModel(wb)
        for name, p in model.named_parameters():
            if "encoder.layers." in name and int(name.split("encoder.layers.")[1].split(".")[0]) >= first:
                p.requires_grad_(True)
        ours = CLIPVisionTowerB200(model, trainable_layers=k)
        model_ckpt = cto.FakeCLIPVisionModel(wb)
        for name, p in model_ckpt.named_parameters():
            p.requires_grad_("encoder.layers." in name and int(name.split("encoder.layers.")[1].split(".")[0]) >= first)
        model_ckpt.gradient_checkpointing = True
        ours_ckpt = CLIPVisionTowerB200(model_ckpt, trainable_layers=k)
        eager_params = [{key: wb[full].clone().requires_grad_(True) for key, full in cto.layer_keys(i).items()} for i in range(first, 23)]

        def loss_of(hs):
            return sum((hs[i].float() * d_outs[i].float()).sum() for i in used)

        def run_a():
            with torch.no_grad():
                h = cto.forward_bf16_eager(wb, x, first)[first]
            hs = {}
            for i in range(first, 23):
                h = eager_layer(h, eager_params[i - first])
                hs[i + 1] = h
            loss_of([hs.get(j) for j in cto.OUT_LAYERS]).backward()
            for p in eager_params:
                for t in p.values():
                    t.grad = None

        def run_b():
            loss_of(ours.hidden_states(x)).backward()
            for p in model.parameters():
                p.grad = None

        def run_d():
            loss_of(ours_ckpt.hidden_states(x)).backward()
            for p in model_ckpt.parameters():
                p.grad = None

        arms = [("A", run_a), ("B", run_b)]
        if hf is not None:
            for m in (hf, hf_ckpt):
                for name, p in m.named_parameters():
                    p.requires_grad_("encoder.layers." in name and first <= int(name.split("encoder.layers.")[1].split(".")[0]) < 23)

            def run_hf(m):
                def run():
                    hs = m(pixel_values=x, output_hidden_states=True).hidden_states
                    loss_of([hs[j] for j in cto.OUT_LAYERS]).backward()
                    for p in m.parameters():
                        p.grad = None
                return run

            arms.append(("C", run_hf(hf)))
        arms.append(("D", run_d))
        if hf is not None:
            arms.append(("E", run_hf(hf_ckpt)))
        row = {"trainable_layers": k}
        fitting = []
        for name, fn in arms:
            torch.cuda.empty_cache()
            need = predict_bytes(_lib.lib, name, n, k)
            free = torch.cuda.mem_get_info()[0]
            row[name] = {"predicted_bytes": need, "free_bytes_before": int(free)}
            if need * _MARGIN > free:
                row[name]["does_not_fit"] = f"does not fit: needs {need / 1e9:.1f} GB"
            else:
                fitting.append((name, fn))
        arms = fitting
        times = {name: [] for name, _ in arms}
        mem = {}
        for name, fn in arms:                                       # warm-up, then the peak memory of one step on its own
            fn()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            mem[name] = torch.cuda.max_memory_allocated() - base
            torch.cuda.empty_cache()
        for _ in range(args.rounds):
            for name, fn in arms:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn()
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e))
        fwd_gf, bwd_gf = step_gflop_per_crop(k)
        row.update({"gflop_per_crop_forward": round(fwd_gf, 2), "gflop_per_crop_backward": round(bwd_gf, 2)})
        for name, _ in arms:
            ms = statistics.median(times[name])
            row[name].update({"ms_median": round(ms, 3), "ms_all": [round(t, 3) for t in times[name]],
                              "tflops_algorithmic": round((fwd_gf + bwd_gf) * n / ms, 1), "peak_bytes_above_start": int(mem[name])})
        for a, b in (("B", "A"), ("D", "B"), ("E", "C"), ("D", "E")):
            if a in times and b in times:
                row[f"time_{a}_over_{b}"] = round(row[a]["ms_median"] / row[b]["ms_median"], 3)
                row[f"peak_memory_{a}_over_{b}"] = round(row[a]["peak_bytes_above_start"] / row[b]["peak_bytes_above_start"], 3)
        result["workloads"].append(row)
        del ours, model, ours_ckpt, model_ckpt, eager_params
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
