"""Cost of the gradients w.r.t. the CLIP features in a training step: forward + backward with parameter gradients only, plus dx0,
and plus dx0 and dxm.

    python tools/bench_train_input_grad.py [--crops 64] [--scale 2] [--hidden 4096] [--rounds 30] [--out result.json]

Workload: N = 64 crops, s = 2, hidden 4096 (bench.py's training shape), seeded bf16 features and upstream gradient, a bf16 module.
One step = TokenPackerB200.forward + .backward(grad_out) through autograd, with
    params  input_grad off, features not requiring grad (tp_backward)
    x0      input_grad on, feat requiring grad (tp_backward_inputs with d_x0)
    x0_xm   input_grad on, feat and feat_multi requiring grad (d_x0 and d_xm)
Each step is timed alone with CUDA events (a device synchronise before it), the three variants alternated in every round after
warm-up.  Reports per variant the median, min, max and the quartiles over the rounds, the median increments over ``params``, and
the dxm GEMM's FLOPs (2 R 2048 4096) over the median increment it adds.  The card's name and power limit are read in the same run.
Before timing, the parameter gradients of the three variants are checked to be bit-identical.  Writes nothing but --out.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

VARIANTS = ("params", "x0", "x0_xm")


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--crops", type=int, default=64)
    ap.add_argument("--scale", type=int, default=2)
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_input_grad: needs a CUDA device (there is no CPU measurement)")
    from tokenpacker_b200 import TokenPackerB200
    dev = torch.device("cuda", torch.cuda.current_device())
    n, s, H = args.crops, args.scale, args.hidden
    torch.manual_seed(0)
    m = TokenPackerB200(hidden_size=H, scale_factor=s).to(dev, torch.bfloat16).train()
    g = torch.Generator(device=dev).manual_seed(1)
    x0 = torch.randn(n, 576, 1024, device=dev, generator=g).to(torch.bfloat16)
    xm = torch.randn(n, 576, 4096, device=dev, generator=g).to(torch.bfloat16)
    gout = torch.randn(n, m.num_queries, H, device=dev, generator=g).to(torch.bfloat16)

    def step(variant):
        m.zero_grad(set_to_none=True)
        m.input_grad = variant != "params"
        a0 = x0.detach().requires_grad_(variant != "params")
        am = xm.detach().requires_grad_(variant == "x0_xm")
        m((a0, am)).backward(gout)
        return a0, am

    grads = {}
    for v in VARIANTS:                                                  # warm-up, and the parameter gradients of each variant
        for _ in range(args.warmup):
            a0, am = step(v)
        torch.cuda.synchronize()
        grads[v] = [p.grad.clone() for p in m.parameters()]
        assert (a0.grad is not None) == (v != "params") and (am.grad is not None) == (v == "x0_xm")
        for t in (a0.grad, am.grad):
            assert t is None or bool(torch.isfinite(t.float()).all())
    for v in VARIANTS[1:]:
        assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(grads["params"], grads[v])), v
    del grads

    times = {v: [] for v in VARIANTS}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for v in VARIANTS:
            torch.cuda.synchronize()
            e0.record()
            step(v)
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1))

    def stats(xs):
        q = statistics.quantiles(xs, n=4)
        return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "q1": q[0], "q3": q[2]}
    med = {v: statistics.median(times[v]) for v in VARIANTS}
    R = n * 576
    dxm_flop = 2.0 * R * 2048 * 4096
    inc_xm = med["x0_xm"] - med["x0"]
    rec = {"what": f"TokenPackerB200 forward + backward, N={n} s={s} H={H}, bf16 module, autograd", "card": card(dev),
           "rounds": args.rounds, "ms": {v: stats(times[v]) for v in VARIANTS},
           "median_increment_ms": {"x0": med["x0"] - med["params"], "x0_xm": med["x0_xm"] - med["params"], "xm_over_x0": inc_xm},
           "dxm_gflop": dxm_flop / 1e9,
           "dxm_tflops_from_increment": (dxm_flop / (inc_xm * 1e-3) / 1e12) if inc_xm > 0 else None,
           "param_grads_bit_identical": True, "ms_rounds": times}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
