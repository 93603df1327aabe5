"""Rates of the SM precision probe's legs on cuda:0, next to PyTorch's own GEMMs in the same run.  JSON lines on stdout,
and in <out-dir>/h100_<W>w_precision_rate.jsonl (W: the card's power limit in watts): one line per grid point, then the
PyTorch lines, then the summary line.

Grid: for each leg and each iteration count (`iterations` for the tensor legs, `alu_iterations` for DFMA and HFMA2),
the median over 21 calls of ops / ns (ns: CUDA events around the launches of the leg, so the operand generation, the
per-iteration fold and the compare are inside it) and of the leg's time per call.  PyTorch: torch.matmul on 8192^3 in
float64, in float32 with TF32 allowed (in this process only) and in float16, CUDA events, median of 21 after 3 warm-up
calls.  The card's name, power limit and max SM clock come from a read-only nvidia-smi query in the same run.  Last: 21
calls at the defaults, their wall time, host reference time and per-leg rates."""
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
LEG_NAMES = ["f64", "dfma", "tf32", "f16", "f16acc", "e5m2", "hfma2"]
ALU = {cro.PRECISION_LEG_DFMA, cro.PRECISION_LEG_HFMA2}
G = 8192


def med(xs):
    return sorted(xs)[len(xs) // 2]


def torch_gemms():
    import torch
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = True
    a = torch.randn(G, G, device=dev)
    b = torch.randn(G, G, device=dev)
    cases = {"f64": (a.double(), b.double()), "tf32": (a, b), "f16": (a.half(), b.half())}
    out = {}
    for name, (x, y) in cases.items():
        for _ in range(3):
            torch.matmul(x, y)
        times = []
        for _ in range(ROUNDS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            torch.matmul(x, y)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e6)
        out[name] = int(2 * G ** 3 / med(times))          # flops per ns = GFLOP/s
    return out


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
        ctx.probe_precision(0, iterations=16, alu_iterations=1)     # warm-up: modules loaded, clocks up
        for it in ITERATIONS:
            for leg, name in enumerate(LEG_NAMES):
                rates, ns = [], []
                for _ in range(ROUNDS):
                    kw = dict(alu_iterations=it) if leg in ALU else dict(iterations=it)
                    r, _s, _f = ctx.probe_precision(0, legs=1 << leg, **kw)
                    L = r.leg[leg]
                    assert r.status == cro.OK, (name, it, L.mismatches, L.fold_mismatches)
                    rates.append(L.ops // L.ns)
                    ns.append(L.ns)
                emit({"leg": name, "iterations": it, "rate_median": med(rates), "leg_ns_median": med(ns)})
                best[name] = max(best.get(name, 0), med(rates))
        walls, host_ref, rates, leg_ns = [], [], {n: [] for n in LEG_NAMES}, {n: [] for n in LEG_NAMES}
        for _ in range(ROUNDS):
            t = time.perf_counter_ns()
            r, _s, _f = ctx.probe_precision(0)
            walls.append(time.perf_counter_ns() - t)
            assert r.status == cro.OK
            host_ref.append(r.host_ref_ns)
            for leg, name in enumerate(LEG_NAMES):
                rates[name].append(r.leg[leg].ops // r.leg[leg].ns)
                leg_ns[name].append(r.leg[leg].ns)
        defaults = {"iterations": r.leg[cro.PRECISION_LEG_F64].iterations,
                    "alu_iterations": r.leg[cro.PRECISION_LEG_DFMA].iterations}
        sm_count = r.sm_count
    torch_rates = torch_gemms()
    for name, v in torch_rates.items():
        emit({"torch": name, "shape": [G, G, G], "rate_median": v})
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "sm_count": sm_count, "rounds": ROUNDS,
          "defaults": defaults, "default_call_wall_ns_median": med(walls), "host_ref_ns_median": med(host_ref),
          "default_call_rate_median": {n: med(v) for n, v in rates.items()},
          "default_call_leg_ns_median": {n: med(v) for n, v in leg_ns.items()},
          "best_grid_rate": best, "torch_rate": torch_rates,
          "share_of_torch": {k: round(best[k] / torch_rates[k], 3) for k in ("f64", "tf32", "f16")}})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_precision_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
