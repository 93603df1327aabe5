"""Time and rate of the register-file probe on cuda:0.  JSON lines on stdout, and in <out-dir>/h100_<W>w_regfile_rate.jsonl
(W: the card's power limit in watts): one line per iteration count (1, the default and 4096), then the summary.

Per iteration count: the median over --calls calls (in process, cro_probe_regfile) of the time per launch (CUDA events
around the launches, over the rounds), of the whole call's wall time, and of the held bits checked per second (32 * K *
T * 2 * iterations per CTA over the launch time).  The card's name, power limit and max SM clock come from a read-only
nvidia-smi query in the same run."""
import argparse
import importlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")


def med(xs):
    return sorted(xs)[len(xs) // 2]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    ap.add_argument("--calls", type=int, default=9)
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock})
    summary = {}
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as ctx:
        ctx.probe_regfile(0, iterations=4)                                # warm-up: module loaded, clocks up
        for it in (1, 0, 4096):
            per_launch, walls, rates = [], [], []
            for _ in range(args.calls):
                r, _sms, _f = ctx.probe_regfile(0, iterations=it)
                assert r.status == cro.OK, (it, r.status)
                per_launch.append(r.ns / r.rounds)
                walls.append(r.wall_ns)
                rates.append(r.bits_checked / (r.ns / 1e9))
            emit({"iterations": r.iterations, "default": it == 0, "calls": args.calls,
                  "launch_us_median": round(med(per_launch) / 1e3, 1), "wall_ms_median": round(med(walls) / 1e6, 3),
                  "held_bits_per_s_median": round(med(rates)), "rounds": r.rounds, "sms_covered": r.sms_covered,
                  "sm_count": r.sm_count, "num_regs": r.num_regs, "regs_per_sm": r.regs_per_sm,
                  "regs_held_per_sm": r.slots * r.threads})
            summary[str(r.iterations)] = round(med(walls) / 1e6, 3)
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "wall_ms_by_iterations": summary})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_regfile_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
