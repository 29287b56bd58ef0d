"""Training step from the CLIP tower's four hidden states: today's LLaVA input path against forward_hidden_states.

    python tools/bench_train_hidden_states.py [--rounds 20] [--warmup 3] [--out result.json]

Two arms, parameter gradients only (input_grad off, the tower frozen as in every released recipe), bf16 module, s = 2, hidden 4096:
    A  cat     x0 = hs[3][:,1:], xm = torch.cat(hs, -1)[:,1:], proj((x0, xm)), backward: the cat writes feat_multi once and the
               training forward copies the crop-strided view once more (kept until the backward)
    B  layers  proj.forward_hidden_states(hs), backward: the four hidden states read in place
Workloads: N = 64 crops (bench.py's training shape) and the 231-crop HD batch (32 images at patch_num 9: 7.2 crops each on
average, the thumbnail included), each hidden state a [N,577,1024] bf16 tensor as the tower returns it.
Each step is timed alone with CUDA events (a device synchronise before it), the two arms alternated in every round after warm-up.
Per arm: median / min / max / quartiles of the step time and the peak memory allocated during one step above what was allocated
before it (torch.cuda.max_memory_allocated).  Before timing, the output and every parameter gradient of A and B are checked to be
bit-identical.  The card's name and power limit are read (never set) in the same run.  Writes nothing but --out.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_train_input_grad import card  # noqa: E402

ARMS = ("cat", "layers")
WORKLOADS = {"n64": 64, "hd231": 231}


def bench(m, n, rounds, warmup, dev):
    g = torch.Generator(device=dev).manual_seed(n)
    hs = [torch.randn(n, 577, 1024, device=dev, generator=g).to(torch.bfloat16) for _ in range(4)]
    gout = torch.randn(n, m.num_queries, m.hidden_size, device=dev, generator=g).to(torch.bfloat16)

    def step(arm):
        m.zero_grad(set_to_none=True)
        if arm == "cat":
            out = m((hs[3][:, 1:], torch.cat(hs, -1)[:, 1:]))
        else:
            out = m.forward_hidden_states(hs)
        out.backward(gout)
        return out

    ref = {}
    for arm in ARMS:                                                   # warm-up, and the results of each arm
        for _ in range(warmup):
            out = step(arm)
        torch.cuda.synchronize()
        ref[arm] = [out.detach()] + [p.grad.clone() for p in m.parameters()]
        del out
    same = all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(ref["cat"], ref["layers"]))
    assert same, "the two arms differ"
    del ref

    peak = {}
    for arm in ARMS:
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        step(arm)
        torch.cuda.synchronize()
        peak[arm] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20

    times = {a: [] for a in ARMS}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for arm in ARMS:
            torch.cuda.synchronize()
            e0.record()
            step(arm)
            e1.record()
            torch.cuda.synchronize()
            times[arm].append(e0.elapsed_time(e1))

    def stats(xs):
        q = statistics.quantiles(xs, n=4)
        return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "q1": q[0], "q3": q[2]}
    med = {a: statistics.median(times[a]) for a in ARMS}
    return {"crops": n, "ms": {a: stats(times[a]) for a in ARMS}, "median_saving_ms": med["cat"] - med["layers"],
            "median_ratio_layers_over_cat": med["layers"] / med["cat"], "step_peak_mib": peak,
            "peak_saving_mib": peak["cat"] - peak["layers"], "out_and_param_grads_bit_identical": same, "ms_rounds": times}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_hidden_states: needs a CUDA device (there is no CPU measurement)")
    from tokenpacker_b200 import TokenPackerB200
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    m = TokenPackerB200(hidden_size=4096, scale_factor=2).to(dev, torch.bfloat16).train()
    rec = {"what": "TokenPackerB200 forward + backward from four [N,577,1024] bf16 CLIP hidden states, s=2 H=4096, bf16 module, "
                   "parameter gradients only: cat = torch.cat + forward(), layers = forward_hidden_states()",
           "card": card(dev), "rounds": args.rounds,
           "workloads": {k: bench(m, n, args.rounds, args.warmup, dev) for k, n in WORKLOADS.items()}}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
