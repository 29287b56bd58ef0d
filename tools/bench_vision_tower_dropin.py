"""LLaVA's vision-tower seam: three ways to produce (feat, feat_multi) = (hidden_states[23][:, 1:], cat(hidden_states[12, 16, 22,
23], dim=2)[:, 1:]) in the crops' dtype, alone and followed by the projector.

    python tools/bench_vision_tower_dropin.py [--crops 64 231] [--rounds 5] [--out result.json]

Arms, alternated in every round (CUDA events around each call, medians):
  A  transformers' CLIPVisionModel(output_hidden_states=True) + feature_select (clip_encoder.py:28-62): 25 hidden states kept, four
     concatenated, both results cast to the crops' dtype;
  B  CLIPVisionTowerB200.hidden_states + the same [:, 1:] / torch.cat / cast;
  C  the drop-in, tokenpacker_b200.CLIPVisionTower: the tower writes the four hidden states into one [N, 577, 4096] buffer and returns
     views of it (one cast of the whole buffer when the dtypes differ).
Two precisions: the bf16 tower (training) and the fp16 tower fed bf16 crops (evaluation and serving, vision_tower.to(torch.float16)).
Each arm is timed alone and followed by TokenPackerB200.forward (hidden 4096, s = 2), which copies feat into a dense [N, 576, 1024]
operand in every arm.  Peak memory: torch.cuda.max_memory_allocated of one call on its own, above what was allocated before it (the
crops, the weights and the derived caches, built by the warm-up).  Seeded weights at the real shapes (oracle/clip_tower_oracle.py);
transformers is required.  The card's name and power limit are read by the same run and go into the JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_tower_oracle as cto  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--crops", type=int, nargs="+", default=[64, 231])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    import transformers
    from tokenpacker_b200 import CLIPVisionTower, CLIPVisionTowerB200, TokenPackerB200
    dev = "cuda:0"
    w = cto.make_weights(23, seed=11, device=dev)
    cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=24,
                                        image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
    torch.manual_seed(0)
    proj = TokenPackerB200(hidden_size=4096, scale_factor=2).to(dev, torch.bfloat16).eval()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    result = {"bench": "vision_tower_dropin", "gpu": smi, "transformers": transformers.__version__,
              "arm_A": "transformers CLIPVisionModel(output_hidden_states=True) + feature_select + cast",
              "arm_B": "CLIPVisionTowerB200.hidden_states + [:, 1:] / torch.cat + cast", "arm_C": "tokenpacker_b200.CLIPVisionTower",
              "projector": "TokenPackerB200(hidden_size=4096, scale_factor=2).forward((feat, feat_multi))", "workloads": []}
    for tower_dtype in (torch.bfloat16, torch.float16):
        wt = {k: v.to(tower_dtype) for k, v in w.items()}
        hf = transformers.CLIPVisionModel(cfg).to(dev, tower_dtype).eval()
        sd = hf.state_dict()
        sd.update({"vision_model." + k: v for k, v in wt.items()})
        hf.load_state_dict(sd)
        fake = cto.FakeCLIPVisionModel(wt)
        ours = CLIPVisionTowerB200(fake, dtype=tower_dtype)
        dropin = CLIPVisionTower(fake, SimpleNamespace(mm_vision_select_layer=-2, mm_vision_select_feature="patch"))

        def select(hs, dtype):                                      # feature_select on hidden states 12, 16, 22, 23, then .to(images.dtype)
            return hs[3][:, 1:].to(dtype), torch.cat(hs, dim=2)[:, 1:].to(dtype)

        def run_a(x):
            hs = hf(pixel_values=x.to(tower_dtype), output_hidden_states=True).hidden_states      # all 25 kept, as in the reference
            return select([hs[i] for i in cto.OUT_LAYERS], x.dtype)

        arms = {"A": run_a,
                "B": lambda x: select(ours.hidden_states(x), x.dtype),
                "C": lambda x: dropin(x)}
        arms.update({name + "+proj": (lambda f: lambda x: proj(f(x)))(fn) for name, fn in list(arms.items())})
        with torch.no_grad():
            for n in args.crops:
                x = cto.make_images(n, seed=n, device=dev).bfloat16()
                mem = {}
                for name, fn in arms.items():                      # warm-up (derived caches), then one call on its own for its peak
                    fn(x)
                    torch.cuda.synchronize()
                    torch.cuda.empty_cache()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    out = fn(x)
                    torch.cuda.synchronize()
                    mem[name] = torch.cuda.max_memory_allocated() - base
                    del out
                times = {name: [] for name in arms}
                for _ in range(args.rounds):
                    for name, fn in arms.items():
                        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        s.record()
                        out = fn(x)
                        e.record()
                        torch.cuda.synchronize()
                        times[name].append(s.elapsed_time(e))
                        del out
                # C must have B's bits (A differs from both by transformers' own roundings)
                b = arms["B"](x)
                c = arms["C"](x)
                same = all(torch.equal(p.contiguous().view(torch.int16), q.contiguous().view(torch.int16)) for p, q in zip(b, c))
                del b, c
                row = {"tower": str(tower_dtype).replace("torch.", ""), "crops_dtype": "bfloat16", "crops": n, "C_bits_equal_B": same}
                for name in arms:
                    row[name] = {"ms_median": round(statistics.median(times[name]), 3), "ms_all": [round(t, 3) for t in times[name]],
                                 "peak_bytes_above_inputs": int(mem[name])}
                result["workloads"].append(row)
                print(json.dumps(row), file=sys.stderr)
                del x
                torch.cuda.empty_cache()
        del hf, ours, dropin, fake
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
