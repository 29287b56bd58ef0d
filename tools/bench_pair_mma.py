"""The pair GEMM's warpgroup layout against the commit before it: two builds, alternated, each run in its own process.

    python tools/bench_pair_mma.py --base DIR [--new DIR] [--rounds 5] [--out tools/bench_pair_mma_h100.json]

DIR is a checkout of the commit to compare against (for example `git worktree add DIR HEAD~1`); --new defaults to this tree.  Both
trees are built first (make, the library only).  Then, for every round and build (the order of the two builds flips every round):
  - bench.py --no-cpu-baseline --no-extras --dump-outputs: the headline `value`, and stage [1]'s shape alone from its `roofline`
    record (M = 36864, N = 2048, K = 4096, bias + GELU, 10 launches; the kernel choice sends that single GEMM to the one-CTA
    kernel); the dumped output's sha256 is compared across builds
  - the same shape on the pair kernel alone (TP_GEMM_MODE=2, 20 launches after 3 warm-ups, CUDA events)
  - bench.py --workload train: forward + backward step time
  - tools/bench_clip_tower.py --crops 64: the CLIP tower's time (arm B; arm A and the whole path are not used here)
The card's name, power limit and SM clocks are read with nvidia-smi before and after the rounds.  Medians and min-max spreads per build.
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def smi():
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def run_json(tree, args, **extra_env):
    env = dict(os.environ, PYTHONPATH=tree, **extra_env)
    r = subprocess.run([sys.executable] + args, cwd=tree, env=env, capture_output=True, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"{args} in {tree} failed ({r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    return json.loads(lines[-1])


# stage [1]'s shape (k/v_proj.0: M = 36864, N = 2048, K = 4096, bias + GELU) forced onto the pair kernel; seeded inputs
PAIR_ALONE = r"""
import json, torch
from tokenpacker_b200.kernels import gemm_bf16
g = torch.Generator(device="cuda").manual_seed(0)
m, n, k = 36864, 2048, 4096
a = torch.randn(m, k, device="cuda", generator=g).bfloat16()
w = (torch.randn(n, k, device="cuda", generator=g) * 0.02).bfloat16()
b = torch.randn(n, device="cuda", generator=g) * 0.1
c = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
for _ in range(3):
    gemm_bf16(a, w, bias=b, gelu=True, out=c)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 20
e0.record()
for _ in range(reps):
    gemm_bf16(a, w, bias=b, gelu=True, out=c)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
print(json.dumps({"ms": ms, "tflops": 2.0 * m * n * k / (ms * 1e-3) / 1e12}))
"""


def one_round(tree, steps, warmup):
    with tempfile.TemporaryDirectory() as d:
        head = run_json(tree, ["bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--no-cpu-baseline", "--no-extras",
                               "--dump-outputs", d])
        with open(os.path.join(d, "projector_out.npy"), "rb") as f:
            digest = hashlib.sha256(f.read()).hexdigest()
    pair = run_json(tree, ["-c", PAIR_ALONE], TP_GEMM_MODE="2")
    train = run_json(tree, ["bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--workload", "train"])
    tower = run_json(tree, ["tools/bench_clip_tower.py", "--crops", "64", "--rounds", "3", "--err-crops", "1", "--path-crops", "8"])
    roof = head["roofline"]
    return {"value": head["value"], "ms_per_step": head["ms_per_step"], "stage1_ms": roof["ms_per_launch"], "stage1_tflops": roof["achieved"],
            "stage1_pair_ms": pair["ms"], "stage1_pair_tflops": pair["tflops"],
            "clocks": head.get("clocks"), "train_ms": train["value"], "tower64_ms": tower["workloads"][0]["B"]["ms_median"], "dump_sha256": digest}


def summary(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "spread": max(xs) - min(xs), "all": xs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="tree of the commit to compare against")
    ap.add_argument("--new", default=ROOT)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    trees = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new)}
    for tree in trees.values():
        subprocess.run(["make", "-C", os.path.join(tree, "tokenpacker_b200", "csrc"), "../libtokenpacker_b200.so"], check=True,
                       stdout=subprocess.DEVNULL)
    result = {"bench": "pair_mma_ab", "gpu_before": smi(), "rounds": []}
    for i in range(args.rounds):
        order = ("base", "new") if i % 2 == 0 else ("new", "base")
        rnd = {name: one_round(trees[name], args.steps, args.warmup) for name in order}
        rnd["order"] = list(order)
        result["rounds"].append(rnd)
        print(json.dumps({"round": i, **{k: {m: rnd[k][m] for m in ("value", "stage1_ms", "stage1_pair_ms", "train_ms", "tower64_ms")} for k in trees}}), flush=True)
    result["gpu_after"] = smi()
    for name in trees:
        result[name] = {m: summary([r[name][m] for r in result["rounds"]])
                        for m in ("value", "ms_per_step", "stage1_ms", "stage1_tflops", "stage1_pair_ms", "stage1_pair_tflops", "train_ms",
                                  "tower64_ms")}
    result["outputs_identical"] = all(r["base"]["dump_sha256"] == r["new"]["dump_sha256"] for r in result["rounds"])
    result["value_gain"] = result["new"]["value"]["median"] / result["base"]["value"]["median"] - 1.0
    result["stage1_gain"] = result["base"]["stage1_ms"]["median"] / result["new"]["stage1_ms"]["median"] - 1.0
    result["stage1_pair_gain"] = result["base"]["stage1_pair_ms"]["median"] / result["new"]["stage1_pair_ms"]["median"] - 1.0
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
