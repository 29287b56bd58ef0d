"""The pair GEMM's tile epilogue against the commit before it: two builds, alternated, each run in its own process.

    python tools/bench_epilogue.py --base DIR [--new DIR] [--rounds 5] [--out tools/bench_epilogue_h100.json]
    python tools/bench_epilogue.py --premise [--new DIR]         (the K sweep alone, on one tree)

A round takes about four minutes on an H100; --resume JSON continues a run that was cut short from its last written --out.

DIR is a checkout of the commit to compare against (for example `git worktree add DIR HEAD~1`); --new defaults to this tree.  Both
trees are built first (make: the library and the test-hook library).  Then, for every round and build (the order of the two builds
flips every round):
  - bench.py --no-cpu-baseline --no-extras --dump-outputs: the headline `value` and `ms_per_step`; the dumped output's sha256 is
    compared across builds
  - bench.py --workload train: forward + backward step time
  - the K sweep: the pair kernel alone (TP_GEMM_MODE=2) at M = 36864, N = 1024 (576 tiles of 256 x 256: 9 tiles per CTA pair on a
    132-SM H100, the last wave 48 of 66 pairs), K = 256 .. 4096, once per epilogue kind (bias; bias + GELU; LayerNorm fold; bias +
    GELU + row statistics; dual), launched through the test-hook library's tpt_gemm_group with the items of
    tests/test_gemm_engine_gpu.py.  A least-squares line of time per tile against K: its intercept is the fixed cost of a tile that
    does not shrink with K — the epilogue, the column-vector staging, the ramp of the mainloop — and its slope the mainloop's
    cost per unit of K.
  - tools/bench_clip_tower.py --crops 64: the CLIP tower's time (arm B)
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
KS = (256, 512, 1024, 2048, 4096)
KINDS = ("bias", "gelu", "ln", "stats", "dual")


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


# the K sweep of one tree, in its own process (TP_GEMM_MODE=2: every item on the pair kernel); seeded inputs
SWEEP = r"""
import json, sys, torch
sys.path.insert(0, "tests")
from test_gemm_engine_gpu import Hooks, Item, PAIR
M, N = 36864, 1024
KW = {"bias": dict(bias=True), "gelu": dict(bias=True, gelu=True), "ln": dict(bias=True, ln=True),
      "stats": dict(bias=True, gelu=True, stats=True), "dual": dict(bias=True, gelu=True, dual=True)}
hk = Hooks()
pairs = hk.sms // 2
tiles = (M // 256) * (N // 256)
waves = -(-tiles // pairs)
out = {"M": M, "N": N, "tiles": tiles, "pairs": pairs, "tiles_per_pair": waves, "kinds": {}}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for kind in %(kinds)r:
    rows = []
    for k in %(ks)r:
        it = Item(0, M, N, k, seed=k, **KW[kind])
        assert hk.choice(it) == PAIR
        for _ in range(3):
            assert hk.group([it]) == 0
        torch.cuda.synchronize()
        reps = 20
        e0.record()
        for _ in range(reps):
            hk.group([it])
        e1.record()
        torch.cuda.synchronize()
        rows.append({"K": k, "ms": e0.elapsed_time(e1) / reps})
        del it
        torch.cuda.empty_cache()
    # time per tile (per CTA pair: `waves` tiles in sequence) = intercept + slope * K, least squares
    xs = [r["K"] for r in rows]
    ys = [r["ms"] * 1e3 / waves for r in rows]
    mx, my = sum(xs) / len(xs), sum(ys) / len(ys)
    slope = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sum((x - mx) ** 2 for x in xs)
    out["kinds"][kind] = {"points": rows, "us_per_tile_intercept": my - slope * mx, "us_per_tile_per_1024k": slope * 1024}
print(json.dumps(out))
"""


def sweep(tree):
    return run_json(tree, ["-c", SWEEP % {"kinds": KINDS, "ks": KS}], TP_GEMM_MODE="2")


def one_round(tree, steps, warmup):
    with tempfile.TemporaryDirectory() as d:
        head = run_json(tree, ["bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--no-cpu-baseline", "--no-extras",
                               "--dump-outputs", d])
        with open(os.path.join(d, "projector_out.npy"), "rb") as f:
            digest = hashlib.sha256(f.read()).hexdigest()
    train = run_json(tree, ["bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--workload", "train"])
    sw = sweep(tree)
    tower = run_json(tree, ["tools/bench_clip_tower.py", "--crops", "64", "--rounds", "3", "--err-crops", "1", "--path-crops", "8"])
    rec = {"value": head["value"], "ms_per_step": head["ms_per_step"], "clocks": head.get("clocks"), "train_ms": train["value"],
           "tower64_ms": tower["workloads"][0]["B"]["ms_median"], "dump_sha256": digest, "sweep": sw}
    for kind, r in sw["kinds"].items():
        rec[f"intercept_us_{kind}"] = r["us_per_tile_intercept"]
    return rec


def summary(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "spread": max(xs) - min(xs), "all": xs}


def build(tree):
    subprocess.run(["make", "-C", os.path.join(tree, "tokenpacker_b200", "csrc"), "../libtokenpacker_b200.so",
                    "../libtokenpacker_b200_testhooks.so"], check=True, stdout=subprocess.DEVNULL)


def write(result, path):
    line = json.dumps(result)
    if path:
        with open(path, "w") as f:
            f.write(line + "\n")
    else:
        print(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="tree of the commit to compare against")
    ap.add_argument("--new", default=ROOT)
    ap.add_argument("--premise", action="store_true", help="only the K sweep, on --new")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--resume", metavar="JSON", default=None, help="an earlier, cut-short --out of the same trees: run the missing rounds")
    args = ap.parse_args()
    if args.premise:
        tree = os.path.abspath(args.new)
        build(tree)
        write({"bench": "epilogue_premise", "gpu_before": smi(), "sweep": sweep(tree), "gpu_after": smi()}, args.out)
        return
    if not args.base:
        ap.error("--base is required unless --premise")
    trees = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new)}
    for tree in trees.values():
        build(tree)
    metrics = ("value", "ms_per_step", "train_ms", "tower64_ms") + tuple(f"intercept_us_{k}" for k in KINDS)
    result = {"bench": "epilogue_ab", "gpu_before": smi(), "rounds": []}
    if args.resume:
        with open(args.resume) as f:
            result = json.load(f)
        result["gpu_resumed"] = result.get("gpu_resumed", []) + [smi()]
    for i in range(len(result["rounds"]), args.rounds):
        order = ("base", "new") if i % 2 == 0 else ("new", "base")
        rnd = {name: one_round(trees[name], args.steps, args.warmup) for name in order}
        rnd["order"] = list(order)
        result["rounds"].append(rnd)
        print(json.dumps({"round": i, **{k: {m: rnd[k][m] for m in metrics} for k in trees}}), flush=True)
        summarize(result, trees, metrics)
        write(result, args.out)           # after every round: a cut-short run keeps the rounds it finished
    result["gpu_after"] = smi()
    summarize(result, trees, metrics)
    write(result, args.out)


def summarize(result, trees, metrics):
    for name in trees:
        result[name] = {m: summary([r[name][m] for r in result["rounds"]]) for m in metrics}
    result["outputs_identical"] = all(r["base"]["dump_sha256"] == r["new"]["dump_sha256"] for r in result["rounds"])
    result["value_gain"] = result["new"]["value"]["median"] / result["base"]["value"]["median"] - 1.0
    result["train_gain"] = result["base"]["train_ms"]["median"] / result["new"]["train_ms"]["median"] - 1.0
    result["tower64_gain"] = result["base"]["tower64_ms"]["median"] / result["new"]["tower64_ms"]["median"] - 1.0


if __name__ == "__main__":
    main()
