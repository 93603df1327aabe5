"""Rates of the SM warp-MMA probe's legs on cuda:0, with PyTorch's dense GEMM in the same run as context.  JSON lines on
stdout, and in <out-dir>/h100_<W>w_warpmma_rate.jsonl (W: the card's power limit in watts): one line per grid point,
then the PyTorch line, then the summary line.

Grid: for each leg and iteration count, the median over 21 calls of ops / ns (ns: CUDA events around the launches of
the leg, so the operand generation, the per-iteration fold and the compare are inside it) and of the leg's time per
call.  Ops are 2 M N K per iteration (MOVE: the M N elements it moves).  PyTorch: torch.matmul of two float16 8192 x
8192 matrices, CUDA events, median of 21 after 3 warm-up calls; it runs on wgmma, not mma.sync, so it is context, not a
target.  The card's name, power limit and max SM clock come from a read-only nvidia-smi query in the same run.  Last:
21 calls at the defaults, their wall time, host reference time and per-leg rates."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")

ROUNDS = 21
ITERATIONS = [16, 64, 256, 1024, 4096]
LEG_NAMES = ["s8", "f16", "bf16", "tf32", "f16acc", "move"]
G = 8192


def med(xs):
    return sorted(xs)[len(xs) // 2]


def torch_matmul():
    import torch
    a = torch.randint(-3, 4, (G, G), device="cuda:0").half()
    b = torch.randint(-3, 4, (G, G), device="cuda:0").half()
    for _ in range(3):
        torch.matmul(a, b)
    times = []
    for _ in range(ROUNDS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.matmul(a, b)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e6)
    return {"torch": "matmul", "dtype": "f16", "shape": [G, G, G], "rate_median": int(2 * G ** 3 / med(times)),
            "path": "wgmma (context, not a target)"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    best = {}
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0]) as ctx:
        ctx.probe_warpmma(0, iterations=16)                         # warm-up: modules loaded, clocks up
        for it in ITERATIONS:
            for leg, name in enumerate(LEG_NAMES):
                rates, ns = [], []
                for _ in range(ROUNDS):
                    r, _s, _f = ctx.probe_warpmma(0, legs=1 << leg, iterations=it)
                    L = r.leg[leg]
                    assert r.status == cro.OK, (name, it, L.mismatches, L.fold_mismatches)
                    rates.append(L.ops // L.ns)
                    ns.append(L.ns)
                emit({"leg": name, "iterations": it, "rate_median": med(rates), "leg_ns_median": med(ns)})
                best[name] = max(best.get(name, 0), med(rates))
        walls, host_ref, rates, leg_ns = [], [], {n: [] for n in LEG_NAMES}, {n: [] for n in LEG_NAMES}
        for _ in range(ROUNDS):
            t = time.perf_counter_ns()
            r, _s, _f = ctx.probe_warpmma(0)
            walls.append(time.perf_counter_ns() - t)
            assert r.status == cro.OK
            host_ref.append(r.host_ref_ns)
            for leg, name in enumerate(LEG_NAMES):
                rates[name].append(r.leg[leg].ops // r.leg[leg].ns)
                leg_ns[name].append(r.leg[leg].ns)
        iterations, sm_count = r.leg[0].iterations, r.sm_count
    emit(torch_matmul())
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "sm_count": sm_count, "rounds": ROUNDS,
          "rate_unit": "GOP/s (s8) or GFLOP/s: 2 M N K per ns; move: G elements/s",
          "defaults": {"iterations": iterations}, "default_call_wall_ns_median": med(walls),
          "host_ref_ns_median": med(host_ref), "default_call_rate_median": {n: med(v) for n, v in rates.items()},
          "default_call_leg_ns_median": {n: med(v) for n, v in leg_ns.items()}, "best_grid_rate": best})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_warpmma_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
