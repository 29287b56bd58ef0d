"""Per-tile timeline of the fused forward: where a tile of the persistent pair kernel spends its time, stage by stage.

    python tools/bench_tile_timeline.py [--tree DIR] [--crops 64] [--runs 5] [--out tools/bench_tile_timeline_h100.json]

Copies the native sources of DIR (default: this tree) to a temporary directory, adds the timeline to the pair kernel there (PATCHES
below: the library itself has no such switch, and its kernels stay as they are), builds tools/csrc/tp_tile_timeline.cu — the
product translation unit plus a setter for the timeline buffer, compiled like the test-hook library — and runs bench.py's
flagship forward (configs[1]: s = 2, H = 4096, N crops) through it.  Lane 0 of epilogue warp 0 of every CTA records %globaltimer at the start of each tile's mainloop wait, the end of
its mainloop (for KV-attention tiles also the end of phase K's mainloop and of phase K's epilogue) and the end of its epilogue.
Per tile:
    mainloop  = time between the mainloop wait's start and the last wgmma's retirement (KV tiles: phase K's plus phase V's)
    tile      = start of the CTA's next tile minus start of this one (the CTA's last tile: end of its epilogue)
    fixed     = tile - mainloop: epilogue(s), the column-vector staging and the barriers around them; the tensor pipe idles
Reported per stage ([1], [2], [3]q, KV, [4], [5]): medians over every tile of every run, in microseconds.  The card's name and
power limit are read in the same run.  Writes one JSON line (to --out, or stdout).
"""
import argparse
import ctypes as C
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# the Makefile's NVCCFLAGS (tokenpacker_b200/csrc/Makefile)
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden",
         "--expt-relaxed-constexpr", "-shared", "-cudart", "static"]
# problems of the fused forward's launch, in group order (tp_api.cu, forward_impl)
STAGES = ["[1]", "[2]", "[2]", "[2]", "[3]q", "KV", "[4]", "[5]"]


def smi():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


# (file, anchor, replacement): every anchor must occur exactly `count` times.  Lane 0 of epilogue warp 0 of every CTA writes the
# record of each of its tiles: [0] start of the mainloop wait  [1] end of the (last) mainloop  [2] end of the epilogue
# [3] KV-attention tiles: end of phase K's epilogue  [4] KV-attention tiles: end of phase K's mainloop  [5] problem  [6] tile
REC = "if (tl_rec != nullptr) tl_rec[%d] = globaltimer();"
PATCHES = [
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "  FrontWork front;\n};\n", 1,
     "  FrontWork front;\n  unsigned long long* timeline;\n};\n"
     "constexpr int kTimelineSlots = 8;\nconstexpr int kTimelineTiles = 256;\n"
     "__device__ __forceinline__ unsigned long long globaltimer() {\n"
     "  unsigned long long t;\n  asm volatile(\"mov.u64 %0, %globaltimer;\" : \"=l\"(t));\n  return t;\n}\n"),
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "      float* s_col = s_col_base;\n", 1,
     "      float* s_col = s_col_base;\n"
     "      unsigned long long* tl_rec = nullptr;\n"
     "      if (grp.timeline != nullptr && e == 0 && lane == 0 && (tile - pair_idx) / num_pairs < kTimelineTiles) {\n"
     "        tl_rec = grp.timeline + (static_cast<long long>(blockIdx.x) * kTimelineTiles + (tile - pair_idx) / num_pairs) * kTimelineSlots;\n"
     "        tl_rec[5] = static_cast<unsigned long long>(t.pr - grp.p);\n"
     "        tl_rec[6] = static_cast<unsigned long long>(tile);\n"
     "      }\n"),
    # KV-attention tiles
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "        mbar_wait(&full_bar[stage], phase);\n", 1, REC % 0 + "\n        mbar_wait(&full_bar[stage], phase);\n"),
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "        float mu, rstd;", 1, REC % 4 + "\n        float mu, rstd;"),
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "// everyone is done reading phase K's vectors\n", 1, "// everyone is done reading phase K's vectors\n" + REC % 3 + "\n"),
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "        col_vectors_ready();\n        attn_pv(", 1, REC % 1 + "\n        col_vectors_ready();\n        attn_pv("),
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "        if (at.done_counter != nullptr) {", 1, REC % 2 + "\n        if (at.done_counter != nullptr) {"),
    # the other tiles
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "      const int n_kb = t.kb1 - t.kb0;\n", 1, "      const int n_kb = t.kb1 - t.kb0;\n" + REC % 0 + "\n"),
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "      col_vectors_ready();\n      if (pr.use_tma_store) {", 1, REC % 1 + "\n      col_vectors_ready();\n      if (pr.use_tma_store) {"),
    ("tokenpacker_b200/csrc/tp_gemm.cuh", "static_cast<long long>(t.split) * pr.c_split_stride);\n      }\n", 1,
     "static_cast<long long>(t.split) * pr.c_split_stride);\n      }\n" + REC % 2 + "\n"),
    # the launches take the buffer the setter of tools/csrc/tp_tile_timeline.cu installed
    ("tokenpacker_b200/csrc/tp_api.cu", "template <bool kTower, bool kF16 = false>\nint launch_built_t(", 1,
     "unsigned long long* g_tile_timeline = nullptr;\ntemplate <bool kTower, bool kF16 = false>\nint launch_built_t("),
    ("tokenpacker_b200/csrc/tp_api.cu", "stream, b.g, b.peers));", 1,
     "stream, [&] { GemmGroup g = b.g; g.timeline = g_tile_timeline; return g; }(), b.peers));"),
    ("tokenpacker_b200/csrc/tp_api.cu", "stream, fp.launch.g, fp.launch.peers));", 1,
     "stream, [&] { fp.launch.g.timeline = g_tile_timeline; return fp.launch.g; }(), fp.launch.peers));"),
]


def build(tree, out_dir):
    src = os.path.join(out_dir, "src")
    for d in ("tokenpacker_b200/csrc", "include", "tools/csrc"):
        shutil.copytree(os.path.join(tree, d), os.path.join(src, d))
    for rel, anchor, count, repl in PATCHES:
        path = os.path.join(src, rel)
        text = open(path).read()
        assert text.count(anchor) == count, (rel, anchor, text.count(anchor))
        with open(path, "w") as f:
            f.write(text.replace(anchor, repl))
    so = os.path.join(out_dir, "libtokenpacker_b200_timeline.so")
    subprocess.run([NVCC] + FLAGS + ["-o", so, os.path.join(src, "tools", "csrc", "tp_tile_timeline.cu")], check=True,
                   stdout=subprocess.DEVNULL)
    return so


def med(xs):
    return statistics.median(xs) if xs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=ROOT, help="source tree to build the timeline library from")
    ap.add_argument("--crops", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from tokenpacker_b200 import TokenPackerB200, synthetic as syn
    assert torch.cuda.is_available(), "the timeline needs an H100"
    gpu_before = smi()
    s, H, n = 2, 4096, args.crops
    with tempfile.TemporaryDirectory() as d:
        lib = C.CDLL(build(os.path.abspath(args.tree), d))
    lib.tp_workspace_bytes.restype = C.c_size_t
    lib.tp_workspace_bytes.argtypes = [C.c_int64, C.c_int, C.c_int]
    lib.tp_forward.restype = C.c_int
    lib.tp_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.tpl_set_timeline.argtypes = [C.c_void_p]
    shape = (C.c_int64 * 2)()
    assert lib.tpl_timeline_shape(shape) == 0
    per_cta, slots = int(shape[0]), int(shape[1])

    dev = torch.device("cuda:0")
    m = TokenPackerB200(hidden_size=H, scale_factor=s)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in syn.synthetic_state_dict(H, seed=0).items()})
    m = m.to(dev, torch.bfloat16).eval()
    packed = m._packed_weights(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    x0 = torch.randn((n, 576, 1024), device=dev, generator=g).to(torch.bfloat16)
    xm = torch.randn((n, 576, 4096), device=dev, generator=g).to(torch.bfloat16)
    out = torch.empty((n * (24 // s) ** 2, H), device=dev, dtype=torch.bfloat16)
    wsb = lib.tp_workspace_bytes(n, s, H)
    ws = torch.empty(wsb, device=dev, dtype=torch.uint8)
    n_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tl = torch.zeros((n_sms, per_cta, slots), device=dev, dtype=torch.int64)
    stream = torch.cuda.current_stream().cuda_stream

    def fwd():
        st = lib.tp_forward(packed.data_ptr(), x0.data_ptr(), xm.data_ptr(), n, 576 * 1024, 576 * 4096, s, H, out.data_ptr(), None,
                            ws.data_ptr(), wsb, stream)
        assert st == 0, st

    for _ in range(5):
        fwd()
    torch.cuda.synchronize()
    rows = {k: {"mainloop": [], "fixed": [], "tile": [], "epi_k": [], "epi_v": []} for k in dict.fromkeys(STAGES)}
    lib.tpl_set_timeline(C.c_void_p(tl.data_ptr()))
    for _ in range(args.runs):
        tl.zero_()
        fwd()
        torch.cuda.synchronize()
        rec = tl.cpu().tolist()
        for cta in rec:
            used = [r for r in cta if r[0] != 0]
            for i, r in enumerate(used):
                stage = STAGES[r[5]]
                end = used[i + 1][0] if i + 1 < len(used) else r[2]
                if stage == "KV":
                    main = (r[4] - r[0]) + (r[1] - r[3])
                    rows[stage]["epi_k"].append((r[3] - r[4]) / 1e3)
                    rows[stage]["epi_v"].append((r[2] - r[1]) / 1e3)
                else:
                    main = r[1] - r[0]
                rows[stage]["mainloop"].append(main / 1e3)
                rows[stage]["tile"].append((end - r[0]) / 1e3)
                rows[stage]["fixed"].append((end - r[0] - main) / 1e3)
    lib.tpl_set_timeline(None)
    result = {"bench": "tile_timeline", "tree": os.path.relpath(os.path.abspath(args.tree), ROOT) if args.tree != ROOT else ".",
              "workload": f"configs[1] forward: s={s}, H={H}, N={n} crops, one launch of tp_gemm2_kernel", "runs": args.runs,
              "gpu_before": gpu_before, "stages": {}}
    for stage, r in rows.items():
        e = {"records_per_run": len(r["tile"]) // args.runs, "mainloop_us_median": med(r["mainloop"]), "fixed_us_median": med(r["fixed"]),
             "tile_us_median": med(r["tile"])}
        if stage == "KV":
            e["epilogue_k_us_median"] = med(r["epi_k"])
            e["epilogue_v_us_median"] = med(r["epi_v"])
        result["stages"][stage] = e
    result["gpu_after"] = smi()
    line = json.dumps(result)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
