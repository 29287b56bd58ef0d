"""The KV-attention tiles' fragment epilogue against the commit before it: two builds, alternated, each run in its own process.

    python tools/bench_kv_epilogue.py --base DIR [--new DIR] [--rounds 5] [--parts headline,train,tower] [--out JSON]

DIR is a checkout of the commit to compare against (for example `git worktree add DIR HEAD~1`); --new defaults to this tree.  Both
trees' libraries are built first (make).  Then, for every round and build (the order of the two builds flips every round), the
--parts selected of:
  - bench.py --no-cpu-baseline --no-extras --dump-outputs: the headline `value` and `ms_per_step`
  - bench.py --workload train: forward + backward step time
  - tools/bench_clip_tower.py --crops 64: the CLIP tower's time (arm B)
The dumped outputs of the two builds are compared (max-abs and rel-RMS of new against base: the KV-attention tiles sum in another
order, so the last bits of ctx and what follows it may differ).  The card's name, power limit and SM clocks are read with
nvidia-smi before and after the rounds.  Medians and min-max spreads per build.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_epilogue import ROOT, run_json, smi, summary, write  # noqa: E402

METRICS = {"headline": ("value", "ms_per_step"), "train": ("train_ms",), "tower": ("tower64_ms",)}


def build(tree):
    subprocess.run(["make", "-C", os.path.join(tree, "tokenpacker_b200", "csrc"), "../libtokenpacker_b200.so"], check=True, stdout=subprocess.DEVNULL)


def one_round(tree, parts, steps, warmup):
    rec, out = {}, None
    if "headline" in parts:
        with tempfile.TemporaryDirectory() as d:
            head = run_json(tree, ["bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--no-cpu-baseline",
                                   "--no-extras", "--dump-outputs", d])
            out = np.load(os.path.join(d, "projector_out.npy")).astype(np.float64)
        rec.update(value=head["value"], ms_per_step=head["ms_per_step"], clocks=head.get("clocks"))
    if "train" in parts:
        rec["train_ms"] = run_json(tree, ["bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--workload", "train"])["value"]
    if "tower" in parts:
        tower = run_json(tree, ["tools/bench_clip_tower.py", "--crops", "64", "--rounds", "3", "--err-crops", "1", "--path-crops", "8"])
        rec["tower64_ms"] = tower["workloads"][0]["B"]["ms_median"]
    return rec, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="tree of the commit to compare against")
    ap.add_argument("--new", default=ROOT)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--parts", default="headline,train,tower")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    parts = args.parts.split(",")
    metrics = [m for p in parts for m in METRICS[p]]
    trees = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new)}
    for tree in trees.values():
        build(tree)
    result = {"bench": "kv_epilogue_ab", "gpu_before": smi(), "rounds": []}
    outs = {}
    for i in range(args.rounds):
        order = ("base", "new") if i % 2 == 0 else ("new", "base")
        rnd = {}
        for name in order:
            rnd[name], out = one_round(trees[name], parts, args.steps, args.warmup)
            if out is None:
                continue
            if name in outs:
                assert np.array_equal(outs[name], out), f"{name}: the output changed between rounds"
            outs[name] = out
        rnd["order"] = list(order)
        result["rounds"].append(rnd)
        print(json.dumps({"round": i, **{k: {m: rnd[k][m] for m in metrics} for k in trees}}), flush=True)
    result["gpu_after"] = smi()
    for name in trees:
        result[name] = {m: summary([r[name][m] for r in result["rounds"]]) for m in metrics}
    if outs:
        d = outs["new"] - outs["base"]
        result["outputs"] = {"identical": bool(np.array_equal(outs["new"], outs["base"])), "max_abs": float(np.abs(d).max()),
                             "rel_rms": float(np.sqrt((d ** 2).mean() / (outs["base"] ** 2).mean())),
                             "base_max_abs": float(np.abs(outs["base"]).max())}
        result["value_gain"] = result["new"]["value"]["median"] / result["base"]["value"]["median"] - 1.0
        result["value_ranges_disjoint"] = result["new"]["value"]["min"] > result["base"]["value"]["max"]
    for m in ("train_ms", "tower64_ms"):
        if m in metrics:
            result[m.replace("_ms", "_gain")] = result["base"][m]["median"] / result["new"][m]["median"] - 1.0
    write(result, args.out)


if __name__ == "__main__":
    main()
