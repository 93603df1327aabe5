"""Rates of the SM compute probe's legs on cuda:0, next to PyTorch's own GEMMs in the same run.  JSON lines on stdout,
and in <out-dir>/h100_<W>w_compute_rate.jsonl (W: the card's power limit in watts): one line per grid point, then the
PyTorch lines, then the summary line.

Grid: for each tensor leg and each `iterations` value, the median over 21 calls of ops / ns (ns: CUDA events around the
launches of the leg, so the operand generation and the compare are inside it).  Warpgroups per CTA are not a knob: the
tile's M = 128 is two m64 row blocks, one warpgroup each, and a third warpgroup's 128 accumulator registers per thread
do not fit (384 threads x ~208 registers > the SM's 65536).  PyTorch: torch.matmul in bf16, torch._scaled_mm in e4m3
and torch._int_mm in int8 on 8192^3, CUDA events, median of 21 after 3 warm-up calls.  The card's name, power limit and
max SM clock come from a read-only nvidia-smi query in the same run.

--helper: instead, the helper form (cro_probe_compute_uuid) against the in-process form at the default settings:
HELPER_ROUNDS calls of each, alternating, in one context over cuda:0.  One line, appended to --out: the median, least
and largest spawn-to-exit time of the helper, the in-process call's wall time, and per leg the median rate inside the
helper and in process."""
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
TENSOR = [("s8", cro.COMPUTE_LEG_S8), ("bf16", cro.COMPUTE_LEG_BF16), ("e4m3", cro.COMPUTE_LEG_E4M3)]
G = 8192
HELPER_ROUNDS = 9
LEG_NAMES = ["s8", "bf16", "e4m3", "ffma", "imad"]


def med(xs):
    return sorted(xs)[len(xs) // 2]


def torch_gemms():
    import torch
    dev = torch.device("cuda", 0)
    a = torch.randn(G, G, device=dev)
    bt = torch.randn(G, G, device=dev)
    one = torch.tensor(1.0, device=dev)
    cases = {
        "bf16": lambda x=a.bfloat16(), y=bt.bfloat16().t(): torch.matmul(x, y),
        "e4m3": lambda x=a.to(torch.float8_e4m3fn), y=bt.to(torch.float8_e4m3fn).t():
            torch._scaled_mm(x, y, one, one, out_dtype=torch.bfloat16),
        "s8": lambda x=a.clamp(-100, 100).to(torch.int8), y=bt.clamp(-100, 100).to(torch.int8).t(): torch._int_mm(x, y),
    }
    out = {}
    for name, fn in cases.items():
        for _ in range(3):
            fn()
        times = []
        for _ in range(ROUNDS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e6)
        out[name] = int(2 * G ** 3 / med(times))          # ops per ns = GFLOP/s (GOP/s for int8)
    return out


def helper_rates(gpu: str, power: str, clock: str) -> dict:
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0]) as ctx:
        uuid = ctx.own_devices()[0].gpu_uuid.decode()
        ctx.probe_compute(0)                                         # warm-up: modules loaded, clocks up
        cro.probe_compute_uuid(ctx, uuid)
        inproc, helper, spawn, walls = [], [], [], []
        for _ in range(HELPER_ROUNDS):
            t = time.perf_counter_ns()
            r, _s, _f = ctx.probe_compute(0)
            walls.append(time.perf_counter_ns() - t)
            assert r.status == cro.OK
            inproc.append(r)
            r, _s, _f, ns = cro.probe_compute_uuid(ctx, uuid)
            assert r.status == cro.OK
            helper.append(r)
            spawn.append(ns)
    out = {"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "probe": "compute", "rounds": HELPER_ROUNDS,
           "iterations": r.leg[0].iterations, "alu_iterations": r.leg[cro.COMPUTE_LEG_FFMA].iterations,
           "helper_ns_median": med(spawn), "helper_ns_min": min(spawn), "helper_ns_max": max(spawn),
           "in_process_wall_ns_median": med(walls),
           "host_ref_ns_median": {"helper": med([r.host_ref_ns for r in helper]), "in_process": med([r.host_ref_ns for r in inproc])}}
    for leg, name in enumerate(LEG_NAMES):
        out[name + "_rate_median"] = {"helper": med([r.leg[leg].ops // r.leg[leg].ns for r in helper]),
                                      "in_process": med([r.leg[leg].ops // r.leg[leg].ns for r in inproc])}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    ap.add_argument("--helper", action="store_true", help="the helper form against the in-process form")
    ap.add_argument("--out", default=None, help="--helper: append the line to this file")
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    if args.helper:
        emit(helper_rates(gpu, power, clock))
        if args.out:
            with open(args.out, "a") as f:
                f.write("\n".join(lines) + "\n")
        return
    best = {}
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0]) as ctx:
        ctx.probe_compute(0, iterations=16, alu_iterations=1)       # warm-up: modules loaded, clocks up
        for it in ITERATIONS:
            for name, leg in TENSOR:
                rates = []
                for _ in range(ROUNDS):
                    r, _s, _f = ctx.probe_compute(0, iterations=it, legs=1 << leg)
                    assert r.status == cro.OK, (name, it, r.leg[leg].mismatches, r.leg[leg].fold_mismatches)
                    rates.append(r.leg[leg].ops // r.leg[leg].ns)
                emit({"leg": name, "iterations": it, "warpgroups": 2, "rate_median": med(rates)})
                best[name] = max(best.get(name, 0), med(rates))
        walls, host_ref, alu = [], [], {"ffma": [], "imad": []}
        for _ in range(ROUNDS):
            t = time.perf_counter_ns()
            r, _s, _f = ctx.probe_compute(0)
            walls.append(time.perf_counter_ns() - t)
            assert r.status == cro.OK
            host_ref.append(r.host_ref_ns)
            alu["ffma"].append(r.leg[cro.COMPUTE_LEG_FFMA].ops // r.leg[cro.COMPUTE_LEG_FFMA].ns)
            alu["imad"].append(r.leg[cro.COMPUTE_LEG_IMAD].ops // r.leg[cro.COMPUTE_LEG_IMAD].ns)
        default_iterations = r.leg[0].iterations
        default_rates = {name: r.leg[leg].ops // r.leg[leg].ns for name, leg in TENSOR}
        sm_count = r.sm_count
    torch_rates = torch_gemms()
    for name, v in torch_rates.items():
        emit({"torch": name, "shape": [G, G, G], "rate_median": v})
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "sm_count": sm_count, "rounds": ROUNDS,
          "default_iterations": default_iterations, "default_call_wall_ns_median": med(walls),
          "host_ref_ns_median": med(host_ref), "default_call_rates_last": default_rates,
          "ffma_gflops_median": med(alu["ffma"]), "imad_gops_median": med(alu["imad"]),
          "best_grid_rate": best, "torch_rate": torch_rates,
          "share_of_torch": {k: round(best[k] / torch_rates[k], 3) for k in best}})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_compute_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
