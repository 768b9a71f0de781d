"""Where the time of the benchmark's batch step goes: a torch.profiler trace of bench.py's configuration.

    python scripts/trace_batch.py --out DIR [--steps 3] [--warmup 2] [--tree OTHER_TREE]

Runs the plan bench.py times (randn(64^5) fp32 at TT-rank 32, as many tensors per tnb_ttsvd_batch call as bench.py
puts in flight, 4 reserved SMs) for --warmup untimed steps, then --steps steps under torch.profiler with CUDA
activities, synchronised and 50 ms apart so that the steps are told apart by the gaps between their kernels.  Writes
DIR/trace_batch.pt.trace.json (the trace) and DIR/trace_batch.json:
  * kernels: per kernel name, count, total, min / median / max ms over the traced steps;
  * step_ms: per step, the span from its first kernel's start to its last kernel's end;
  * step1_gram_ms: per step, the step-1 Gram of every tensor (the second gram_tc_kernel on each stream), in start order;
  * overlap_ms: per step, the wall time in which a cheb_filter_kernel runs while a gram_tc_kernel or a
    project_tc_kernel runs (separately and together);
  * idle_ms: per step, the time inside the step's span in which no kernel runs;
  * the card's name, power limit and maximum SM clock.
--tree imports the library from a second checkout with its library built (e.g. the parent commit) instead of this one.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FILTER, GRAM, PROJ = "cheb_filter_kernel", "gram_tc_kernel", "project_tc_kernel"


def short_name(name):
    """The kernel's function name without namespace, template arguments or parameters."""
    base = name.split("(")[0].split("<")[0].strip()
    return base.split()[-1].split("::")[-1] if base else name


def union(intervals):
    out = []
    for a, b in sorted(intervals):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def length(intervals):
    return sum(b - a for a, b in intervals)


def intersect(x, y):
    """Intersection of two sorted lists of disjoint intervals."""
    out, i, j = [], 0, 0
    while i < len(x) and j < len(y):
        a, b = max(x[i][0], y[j][0]), min(x[i][1], y[j][1])
        if a < b:
            out.append([a, b])
        if x[i][1] < y[j][1]:
            i += 1
        else:
            j += 1
    return out


def split_steps(kernels, nsteps):
    """Kernels (start-sorted) cut into nsteps groups at the nsteps - 1 widest gaps between the end of everything before
    and the next start."""
    gaps, end = [], kernels[0]["ts"] + kernels[0]["dur"]
    for i in range(1, len(kernels)):
        gaps.append((kernels[i]["ts"] - end, i))
        end = max(end, kernels[i]["ts"] + kernels[i]["dur"])
    cuts = sorted(i for _, i in sorted(gaps, reverse=True)[: nsteps - 1])
    bounds = [0] + cuts + [len(kernels)]
    return [kernels[bounds[k]:bounds[k + 1]] for k in range(nsteps)]


def analyse(kernels):
    """Summary of one step's kernels (times in us in, ms out)."""
    span = [kernels[0]["ts"], max(k["ts"] + k["dur"] for k in kernels)]
    busy = union([[k["ts"], k["ts"] + k["dur"]] for k in kernels])
    by = {n: union([[k["ts"], k["ts"] + k["dur"]] for k in kernels if k["short"] == n]) for n in (FILTER, GRAM, PROJ)}
    per_stream = {}
    for k in kernels:
        if k["short"] == GRAM:
            per_stream.setdefault(k["stream"], []).append(k)
    step1 = sorted((g[1] for g in per_stream.values() if len(g) > 1), key=lambda k: k["ts"])
    return {
        "span_ms": (span[1] - span[0]) / 1e3,
        "idle_ms": (span[1] - span[0] - length(busy)) / 1e3,
        "overlap_ms": {
            "filter_gram": length(intersect(by[FILTER], by[GRAM])) / 1e3,
            "filter_project": length(intersect(by[FILTER], by[PROJ])) / 1e3,
            "filter_gram_or_project": length(intersect(by[FILTER], union(by[GRAM] + by[PROJ]))) / 1e3,
        },
        "step1_gram_ms": [k["dur"] / 1e3 for k in step1],
        "busy_ms": {"filter": length(by[FILTER]) / 1e3, "gram": length(by[GRAM]) / 1e3, "project": length(by[PROJ]) / 1e3},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tree", default=REPO, help="checkout whose built library is traced (default: this one)")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    sys.path.insert(0, os.path.abspath(args.tree))
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    from tntorch_b200 import ops

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    shape, rank = (64,) * 5, 32
    numel = int(np.prod(shape))
    # bench.py's batch: up to 8 tensors, bounded by 60 % of the free memory; 4 reserved SMs when several are in flight
    free_b, _ = torch.cuda.mem_get_info(dev)
    probe = ops.TTSVDBatchPlan(shape, torch.float32, 1, rmax=rank, device=dev, inflight=1)
    per_tensor = numel * 4 + probe.per_tensor_bytes + int(probe.cap) * 4
    del probe
    PB = max(1, min(8, int(0.6 * free_b // per_tensor)))
    ops.set_reserved_sms(4 if PB > 1 else 0)
    Xb = torch.empty((PB,) + shape, device=dev, dtype=torch.float32)
    for b in range(PB):
        g = torch.Generator(device=dev).manual_seed(1234 + b)
        Xb[b].copy_(torch.randn(shape, generator=g, device=dev, dtype=torch.float32))
    plan = ops.TTSVDBatchPlan(shape, torch.float32, PB, rmax=rank, device=dev, inflight=PB)
    for _ in range(args.warmup):
        plan.run(Xb)
    torch.cuda.synchronize()
    wall = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            t0 = time.perf_counter()
            plan.run(Xb)
            torch.cuda.synchronize()
            wall.append((time.perf_counter() - t0) * 1e3)
            time.sleep(0.05)
    trace = os.path.join(args.out, "trace_batch.pt.trace.json")
    prof.export_chrome_trace(trace)
    events = json.load(open(trace))["traceEvents"]
    kernels = sorted(({"name": e["name"], "short": short_name(e["name"]), "ts": float(e["ts"]), "dur": float(e["dur"]),
                       "stream": e.get("args", {}).get("stream")}
                      for e in events if e.get("cat") == "kernel" and e.get("ph") == "X"), key=lambda k: k["ts"])
    if not kernels:
        raise SystemExit("the trace holds no kernels")
    names = {}
    for k in kernels:
        names.setdefault(k["short"], []).append(k["dur"] / 1e3)
    steps = [analyse(s) for s in split_steps(kernels, args.steps)]
    out = {
        "nvidia_smi": smi,
        "config": {"shape": list(shape), "rank": rank, "tensors_per_call": PB, "reserved_sms": 4 if PB > 1 else 0,
                   "tree": os.path.abspath(args.tree), "traced_steps": args.steps},
        "speculative_sweeps_accepted": int(sum(plan.spec)),
        "host_ms_per_step_under_profiler": wall,
        "kernels": {n: {"count": len(d), "total_ms": sum(d), "min_ms": min(d), "median_ms": statistics.median(d),
                        "max_ms": max(d)} for n, d in sorted(names.items(), key=lambda x: -sum(x[1]))},
        "steps": steps,
        "mean": {"span_ms": statistics.mean(s["span_ms"] for s in steps),
                 "idle_ms": statistics.mean(s["idle_ms"] for s in steps),
                 "overlap_filter_gram_or_project_ms": statistics.mean(s["overlap_ms"]["filter_gram_or_project"]
                                                                      for s in steps)},
    }
    json.dump(out, open(os.path.join(args.out, "trace_batch.json"), "w"), indent=1)
    print(json.dumps({k: out[k] for k in ("nvidia_smi", "config", "speculative_sweeps_accepted", "mean")}))
    for i, s in enumerate(steps):
        print(f"step {i}: span {s['span_ms']:.2f} ms, idle {s['idle_ms']:.2f} ms, overlap {s['overlap_ms']}, "
              f"step-1 Grams {[round(x, 2) for x in s['step1_gram_ms']]}")


if __name__ == "__main__":
    main()
