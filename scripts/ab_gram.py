"""A/B of two builds of this repository on one GPU: bench.py alternating between them, their outputs on the same seeded
input, and the TF32 noise floor of their Gram kernels.

    python scripts/ab_gram.py OTHER_TREE --out DIR [--runs 3] [--steps 5] [--warmup 3]

OTHER_TREE is a second checkout with its library already built (e.g. the parent commit).  Every bench.py run is a fresh
process; the JSON written to DIR/ab_gram.json holds, per run, value, ms_per_step, phases_ms.gram_ms, the roofline,
sweep_roofline.single_call_ms and run.speculative_sweeps_accepted, plus the card's name and power limit.  Gram noise:
||G_tf32 - (1 - c) G_fp64||_2 / ||G_fp64||_2 on randn(262144, 2048), c the least-squares truncation bias, for the
row-major Gram and, where the build has it, the Gram of the same matrix stored K-blocked.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gram_noise(tree):
    sys.path.insert(0, tree)
    import torch

    from tntorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randn(262144, 2048, generator=g, device="cuda", dtype=torch.float32)
    grams = {"rowmajor": ops.gram(A, tensorcore=True)}
    if hasattr(ops, "gram_kblocked"):
        grams["kblocked"] = ops.gram_kblocked(ops.to_kblocked(A), *A.shape)
    A64 = A.double()
    ref = A64.T @ A64
    del A64
    out = {"tree": tree}
    for k, G in grams.items():
        c = 1.0 - float((G * ref).sum() / (ref * ref).sum())
        E = G - (1.0 - c) * ref
        noise = float(torch.linalg.matrix_norm(E, ord=2) / torch.linalg.matrix_norm(ref, ord=2))
        out.update({"bias_c" if k == "rowmajor" else f"bias_c_{k}": c,
                    "noise_rel_2norm" if k == "rowmajor" else f"noise_rel_2norm_{k}": noise})
    return out


def bench(tree, args, dump):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup",
           str(args.warmup), "--no-cpu-baseline", "--dump-outputs", dump]
    out = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"{tree}: bench.py failed\n{out.stderr[-4000:]}")
    res = json.loads([line for line in out.stdout.splitlines() if line.startswith("{")][-1])
    ph = res.get("phases_ms", {})
    return {"value": res["value"], "ms_per_step": res.get("ms_per_step"), "gram_ms": ph.get("gram_ms"),
            "factor_ms": ph.get("factor_ms"),
            "roofline": res.get("roofline"), "single_call_ms": res.get("sweep_roofline", {}).get("single_call_ms"),
            "speculative_sweeps_accepted": res.get("run", {}).get("speculative_sweeps_accepted"),
            "ranks": res.get("run", {}).get("ranks"), "rel_error": res.get("rel_error"),
            "rel_error_twin": res.get("rel_error_twin")}


def compare_dumps(a, b):
    import numpy as np

    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    if fa != fb:
        return {"same_files": False}
    shapes_equal, worst = True, 0.0
    for f in fa:
        if not f.endswith(".npy"):
            continue
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        if x.shape != y.shape:
            shapes_equal = False
            continue
        # cores agree up to the sign of each rank-one pair; compare magnitudes
        worst = max(worst, float(np.abs(np.abs(x) - np.abs(y)).max() / max(np.abs(x).max(), 1e-30)))
    return {"same_files": True, "core_shapes_equal": shapes_equal, "max_rel_abs_core_diff": worst}


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--noise":
        print(json.dumps(gram_noise(sys.argv[2])))
        return
    ap = argparse.ArgumentParser()
    ap.add_argument("other")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True, help="directory for ab_gram.json and the dumped cores of both builds")
    args = ap.parse_args()
    other = os.path.abspath(args.other)
    args.out = os.path.abspath(args.out)  # bench.py runs in each tree's directory
    os.makedirs(args.out, exist_ok=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip()
    trees = {"other": other, "this": REPO}
    runs = {k: [] for k in trees}
    for i in range(args.runs):
        for k, tree in trees.items():
            r = bench(tree, args, os.path.join(args.out, f"dump_{k}"))
            runs[k].append(r)
            print(k, i, json.dumps({x: r[x] for x in ("value", "ms_per_step", "gram_ms", "factor_ms", "single_call_ms")}),
                  flush=True)
    noise = {}
    for k, tree in trees.items():
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--noise", tree], capture_output=True, text=True)
        noise[k] = json.loads(out.stdout.strip().splitlines()[-1]) if out.returncode == 0 else {"error": out.stderr[-2000:]}
    summary = {}
    for k in trees:
        v = [r["value"] for r in runs[k]]
        summary[k] = {"median_value": statistics.median(v), "spread": max(v) - min(v),
                      "median_gram_ms": [statistics.median(r["gram_ms"][j] for r in runs[k]) for j in range(2)]
                      if runs[k][0]["gram_ms"] else None,
                      "median_factor_ms": [statistics.median(r["factor_ms"][j] for r in runs[k]) for j in range(2)]
                      if runs[k][0]["factor_ms"] else None}
    result = {"nvidia_smi": smi, "runs": runs, "summary": summary, "noise": noise,
              "dumps": compare_dumps(os.path.join(args.out, "dump_other"), os.path.join(args.out, "dump_this"))}
    json.dump(result, open(os.path.join(args.out, "ab_gram.json"), "w"), indent=1)
    print(json.dumps({"nvidia_smi": smi, "summary": summary, "noise": noise, "dumps": result["dumps"]}))


if __name__ == "__main__":
    main()
