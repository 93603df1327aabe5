"""Rates and wall time of the SRAM probe on cuda:0.  JSON lines on stdout, and in <out-dir>/h100_<W>w_sram_rate.jsonl
(W: the card's power limit in watts): one line per leg, cluster size and iteration count, then the summary.

Per setting: the median over --calls calls (in process, cro_probe_sram) of the leg's time per launch (CUDA events around
the launch, over its rounds) and of its shared-memory rate, bytes read and written by every CTA launched over that
time, in GB/s for the whole GPU and per SM; then the default call's wall time (both legs, the default iterations and
cluster size).  The card's name, power limit and max SM clock come from a read-only nvidia-smi query in the same run."""
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
    ap.add_argument("--iterations", default="1,4,16,64,256", help="comma-separated iteration counts")
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    iters = [int(x) for x in args.iterations.split(",")]
    summary = {}
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as ctx:
        ctx.probe_sram(0, iterations=4)                                  # warm-up: modules loaded, clocks up
        settings = [("smem", cro.SRAM_LEG_SMEM, 0)] + [("dsmem", cro.SRAM_LEG_DSMEM, c) for c in (2, 4, 8)]
        for name, legs, cluster in settings:
            leg = 0 if legs == cro.SRAM_LEG_SMEM else 1
            for it in iters:
                per_launch, gbs, per_sm, rounds, covered = [], [], [], [], []
                for _ in range(args.calls):
                    r, _sms, _f = ctx.probe_sram(0, legs=legs, iterations=it, cluster=cluster)
                    assert r.status == cro.OK, (name, it, r.status)
                    L = r.leg[leg]
                    per_launch.append(L.ns / L.rounds)
                    gbs.append(L.bytes / L.ns)
                    per_sm.append(L.bytes / L.ns / (L.ctas / L.rounds))
                    rounds.append(L.rounds)
                    covered.append(L.sms_covered)
                emit({"leg": name, "cluster": cluster, "iterations": it, "calls": args.calls,
                      "launch_us_median": round(med(per_launch) / 1e3, 1), "gbs_median": round(med(gbs), 1),
                      "gbs_per_sm_median": round(med(per_sm), 1), "rounds_median": med(rounds),
                      "sms_covered_median": med(covered), "bytes_per_sm": r.bytes_per_sm, "sm_count": r.sm_count})
                summary["%s%s_%d" % (name, cluster or "", it)] = round(med(per_launch) / 1e3, 1)
        walls = []
        for _ in range(args.calls):
            r, _sms, _f = ctx.probe_sram(0)
            assert r.status == cro.OK
            walls.append(r.wall_ns)
        emit({"default_call": {"iterations": r.leg[0].iterations, "cluster": r.leg[1].cluster,
                               "local_rounds": r.leg[0].rounds, "network_rounds": r.leg[1].rounds,
                               "network_sms_covered": r.leg[1].sms_covered, "wall_ms_median": round(med(walls) / 1e6, 2)}})
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "launch_us_by_setting": summary})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_sram_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
