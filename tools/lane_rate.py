"""Rates and time of a lane probe (cross-lane, ALU or barrier) on cuda:0.  JSON lines on stdout, and in
<out-dir>/h100_<W>w_<probe>_rate.jsonl (W: the card's power limit in watts): one line per leg and iteration count (16
to 4096; the barrier probe from 1, its CLUSTER leg at clusters of 2), one per default call, then the summary.

Per leg and iteration count: the median over --calls calls (in process, cro_probe_<probe> with that one leg) of the
launch time (CUDA events around the leg's launches, per round) and of the checks per second (ops or rows * 256 *
iterations per CTA over the launch time).  Per default call: the wall time, the host's table build (ALU and barrier)
and each leg's launch time.  The card's name, power limit and max SM clock come from a read-only nvidia-smi query in
the same run.

    python tools/lane_rate.py xlane|alu|barrier [--calls N] [--out-dir DIR]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")

# Per probe: its leg names, the iteration counts each leg runs at, and whether its result has table_ns.
PROBES = {
    "xlane": (["shfl", "vote", "match", "redux", "atoms"], (16, 64, 256, 1024, 4096), False),
    "alu": (["logic", "shift", "iadd", "imul", "float"], (16, 64, 256, 1024, 4096), True),
    "barrier": (["bar", "mbar", "cluster"], (1, 16, 64, 256, 1024, 4096), True),
}


def med(xs):
    return sorted(xs)[len(xs) // 2]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("probe", choices=sorted(PROBES))
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()
    names, grid, has_table = PROBES[args.probe]
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock})
    best = {}
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as ctx:
        probe = getattr(ctx, "probe_" + args.probe)
        probe(0, iterations=4)                                           # warm-up: module loaded, clocks up
        for leg, name in enumerate(names):
            for it in grid:
                per_launch, rates = [], []
                for _ in range(args.calls):
                    r, _sms, _f = probe(0, iterations=it, legs=1 << leg)
                    assert r.status == cro.OK, (leg, it, r.status)
                    per_launch.append(r.leg_ns[leg] / r.rounds)
                    rates.append(r.ops_checked[leg] / (r.leg_ns[leg] / 1e9))
                emit({"leg": name, "iterations": it, "calls": args.calls, "launch_us_median": round(med(per_launch) / 1e3, 1),
                      "us_per_iteration": round(med(per_launch) / 1e3 / it, 3), "ops_checked_per_s_median": round(med(rates)),
                      "rounds": r.rounds, "sms_covered": r.sms_covered, "sm_count": r.sm_count})
                best[name] = max(best.get(name, 0), round(med(rates)))
        walls, legs_ns = [], []
        for _ in range(args.calls):
            r, _sms, _f = probe(0)
            assert r.status == cro.OK, r.status
            walls.append(r.wall_ns)
            legs_ns.append(r.ns)
        default = {"default_iterations": r.iterations, "calls": args.calls, "wall_ms_median": round(med(walls) / 1e6, 3)}
        if has_table:
            default["table_ms"] = round(r.table_ns / 1e6, 3)
        default.update({"launch_ms_median": round(med(legs_ns) / 1e6, 3), "leg_us": [round(x / 1e3, 1) for x in r.leg_ns],
                        "rounds": r.rounds})
        emit(default)
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "best_ops_checked_per_s": best,
          "default_wall_ms": round(med(walls) / 1e6, 3)})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_%s_rate.jsonl" % (watts, args.probe)), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
