"""Training step of the whole CLIP-ViT-L/14-336 tower: forward + backward of CLIPVisionTowerB200(trainable_layers=23,
train_embeddings=True).hidden_states against the same step without the embedding stage and against transformers' CLIPVisionModel with
every parameter unfrozen.

    python tools/bench_clip_tower_embed.py [--rounds 5] [--out result.json]

Workloads: 64 crops without and with gradient checkpointing, 231 crops (a batch of HD crops) with checkpointing only.  Arms:
  layers  CLIPVisionTowerB200(trainable_layers=23): the 23 layers train, the embedding stage gets no gradient
  whole   CLIPVisionTowerB200(trainable_layers=23, train_embeddings=True): every parameter trains
  hf      transformers' CLIPVisionModel in bf16 after requires_grad_(True) (all 24 layers run; post_layernorm unused by the loss)
Checkpointing is the wrapped model's switch (``gradient_checkpointing`` on our fake model, ``gradient_checkpointing_enable()`` on
transformers').  The loss is a fixed weighted sum of hidden states 12 / 16 / 22 / 23.  Seeded weights at the real shapes
(oracle/clip_tower_oracle.py).  Alternated rounds, CUDA events around forward + backward, medians; peak memory of one step above what
was allocated before it.  An arm that runs out of memory is recorded as such.  The card's name, power limit and clocks are read in the
same run.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", nargs="+", default=["64:plain", "64:ckpt", "231:ckpt"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    dev = "cuda:0"
    from tokenpacker_b200 import CLIPVisionTowerB200
    wb = {k: v.bfloat16() for k, v in cto.make_weights(23, seed=11, device=dev).items()}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    result = {"bench": "clip_tower_embed", "gpu_name_powerlimit_maxsmclock_smclock": smi, "rounds": args.rounds, "workloads": []}
    models = {}
    for arm in ("layers", "whole"):
        m = cto.FakeCLIPVisionModel(wb)
        for p in m.parameters():
            p.requires_grad_(True)
        models[arm] = (m, CLIPVisionTowerB200(m, trainable_layers=23, train_embeddings=arm == "whole"))
    hf = None
    try:
        import transformers
        cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=24,
                                            image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
        hf = transformers.CLIPVisionModel(cfg).to(dev, torch.bfloat16).train()
        sd = hf.state_dict()
        sd.update({"vision_model." + k: v for k, v in wb.items()})
        hf.load_state_dict(sd)
        hf.requires_grad_(True)
        del sd
        result["hf"] = f"transformers {transformers.__version__} CLIPVisionModel bf16, every parameter unfrozen"
    except ImportError:
        pass

    for spec in args.workloads:
        n, mode = int(spec.split(":")[0]), spec.split(":")[1]
        ckpt = mode == "ckpt"
        x = cto.make_images(n, seed=n, device=dev).bfloat16()
        g = torch.Generator(device=dev).manual_seed(5)
        d_outs = [(torch.randn(n, 577, 1024, generator=g, device=dev) * 0.1).bfloat16() for _ in cto.OUT_LAYERS]

        def loss_of(hs):
            return sum((h.float() * d.float()).sum() for h, d in zip(hs, d_outs))

        def run_ours(arm):
            model, tower = models[arm]
            model.gradient_checkpointing = ckpt

            def run():
                loss_of(tower.hidden_states(x)).backward()
                for p in model.parameters():
                    p.grad = None
            return run

        def run_hf():
            if ckpt:
                hf.gradient_checkpointing_enable()
            else:
                hf.gradient_checkpointing_disable()
            hs = hf(pixel_values=x, output_hidden_states=True).hidden_states
            loss_of([hs[j] for j in cto.OUT_LAYERS]).backward()
            for p in hf.parameters():
                p.grad = None

        arms = [("layers", run_ours("layers")), ("whole", run_ours("whole"))] + ([("hf", run_hf)] if hf is not None else [])
        row = {"crops": n, "gradient_checkpointing": ckpt}
        fitting, mem = [], {}
        for name, fn in arms:                                       # warm-up, then the peak memory of one step on its own
            torch.cuda.empty_cache()
            try:
                fn()
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                fn()
                torch.cuda.synchronize()
                mem[name] = torch.cuda.max_memory_allocated() - base
                fitting.append((name, fn))
            except torch.OutOfMemoryError:
                row[name] = {"out_of_memory": True}
                for m in [hf] + [m for m, _ in models.values()]:
                    if m is not None:
                        for p in m.parameters():
                            p.grad = None
            torch.cuda.empty_cache()
        times = {name: [] for name, _ in fitting}
        for _ in range(args.rounds):
            for name, fn in fitting:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn()
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e))
        for name, _ in fitting:
            row[name] = {"ms_median": round(statistics.median(times[name]), 3), "ms_all": [round(t, 3) for t in times[name]],
                         "peak_bytes_above_start": int(mem[name])}
        if "whole" in times and "layers" in times:
            row["time_whole_over_layers"] = round(row["whole"]["ms_median"] / row["layers"]["ms_median"], 4)
            row["peak_memory_whole_minus_layers_bytes"] = row["whole"]["peak_bytes_above_start"] - row["layers"]["peak_bytes_above_start"]
        if "whole" in times and "hf" in times:
            row["time_whole_over_hf"] = round(row["whole"]["ms_median"] / row["hf"]["ms_median"], 3)
            row["peak_memory_whole_over_hf"] = round(row["whole"]["peak_bytes_above_start"] / row["hf"]["peak_bytes_above_start"], 3)
        result["workloads"].append(row)
        print(json.dumps(row), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
