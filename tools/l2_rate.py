"""Rates and wall time of the L2 probe on cuda:0.  JSON lines on stdout, and in <out-dir>/h100_<W>w_l2_rate.jsonl (W: the
card's power limit in watts).

Per buffer size and iteration count: the median over --calls calls (in process, cro_probe_l2) of each march element's
rate (its bytes read and written over its %globaltimer window, first CTA start to last CTA end, summed over the
iterations), of the march's CUDA-event time, of the launch gap (event time less the elements' windows, per launch) and
of the call's wall time.  Then the atomic legs at their defaults and at 4 times them (A1 updates per second: two per
counter and CTA; A2 tickets per second), and the locator's HBM read rate (pass 0 over a 1 GiB sweep region) as the
yardstick a buffer that spills out of the L2 falls back to.  The card's name, power limit and max SM clock come from
a read-only nvidia-smi query in the same run."""
import argparse
import importlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")

MIB = 1 << 20
ELEMENT_BYTES = [1, 2, 2, 2, 2, 1]       # times W: M0 writes, M1 .. M4 read and write, M5 reads


def med(xs):
    return sorted(xs)[len(xs) // 2]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    ap.add_argument("--calls", type=int, default=9)
    ap.add_argument("--sizes", default="4,8,16,24,32,48,64,256", help="buffer sizes in MiB, comma-separated")
    ap.add_argument("--iterations", default="1,8,64", help="comma-separated iteration counts")
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    summary = {}
    with cro.ProbeContext(sweep_bytes=512 * MIB, devices=[0], read_sweeps=2, copy_sweeps=1) as ctx:
        ctx.probe_l2(0, bytes=4 * MIB, iterations=4)                    # warm-up: modules loaded, clocks up
        assert ctx.probe_device(0).status == cro.OK
        hbm = []
        for _ in range(args.calls):
            rep, _w = ctx.locate_faults(0, retest=False)
            P = rep.pass_[0]
            assert rep.status == cro.OK and P.mismatches == 0
            hbm.append(P.words_scanned * 8 / P.scan_ns)
        hbm_gbs = round(med(hbm), 1)
        emit({"locator_hbm_read_gbs_median": hbm_gbs, "sweep_bytes": rep.sweep_bytes, "calls": args.calls})
        for mib in [int(x) for x in args.sizes.split(",")]:
            for it in [int(x) for x in args.iterations.split(",")]:
                el_gbs = [[] for _ in range(6)]
                march_ms, gap_us, wall_ms, march_gbs = [], [], [], []
                for _ in range(args.calls):
                    r, _s, _f = ctx.probe_l2(0, bytes=mib * MIB, iterations=it)
                    assert r.status == cro.OK and r.unpublished == 0 and r.fold_ok == 1, (mib, it, r.status, r.verdict)
                    for e in range(6):
                        el_gbs[e].append(ELEMENT_BYTES[e] * r.bytes * it / r.element_ns[e])
                    march_ms.append(r.march_ns / 1e6)
                    gap_us.append((r.march_ns - sum(r.element_ns)) / (6 * it) / 1e3)
                    wall_ms.append(r.wall_ns / 1e6)
                    march_gbs.append(r.march_bytes / r.march_ns)
                row = {"bytes_mib": mib, "iterations": it, "calls": args.calls, "l2_bytes": r.l2_bytes, "sm_count": r.sm_count,
                       "element_gbs_median": [round(med(x), 1) for x in el_gbs], "march_gbs_median": round(med(march_gbs), 1),
                       "march_ms_median": round(med(march_ms), 3), "launch_gap_us_median": round(med(gap_us), 2),
                       "wall_ms_median": round(med(wall_ms), 3)}
                emit(row)
                summary["%dMiB_x%d" % (mib, it)] = {"m1_gbs": row["element_gbs_median"][1], "wall_ms": row["wall_ms_median"]}
        for scale in (1, 4):
            a1, a2 = 65536 * scale, 1024 * scale
            t = {"a1": [], "a1_check": [], "a2": [], "a2_check": []}
            for _ in range(args.calls):
                r, _s, _f = ctx.probe_l2(0, bytes=4 * MIB, iterations=1, a1_counters=a1, a2_counters=a2)
                assert r.status == cro.OK and r.a1_bad == 0 and r.a2_bad == 0 and r.a2_holes == 0
                t["a1"].append(r.a1_ns)
                t["a1_check"].append(r.a1_check_ns)
                t["a2"].append(r.a2_ns)
                t["a2_check"].append(r.a2_check_ns)
            G = r.ctas
            emit({"atomics": {"a1_counters": a1, "a2_counters": a2, "ctas": G, "calls": args.calls,
                              "a1_us_median": round(med(t["a1"]) / 1e3, 1),
                              "a1_gupdates_per_s": round(2 * a1 * G / med(t["a1"]), 2),
                              "a1_check_us_median": round(med(t["a1_check"]) / 1e3, 1),
                              "a2_us_median": round(med(t["a2"]) / 1e3, 1),
                              "a2_gtickets_per_s": round(32 * G * a2 / med(t["a2"]), 2),
                              "a2_check_us_median": round(med(t["a2_check"]) / 1e3, 1)}})
        walls = []
        for _ in range(args.calls):
            r, _s, _f = ctx.probe_l2(0)
            assert r.status == cro.OK
            walls.append(r.wall_ns)
        emit({"default_call": {"bytes": r.bytes, "iterations": r.iterations, "a1_counters": r.a1_counters,
                               "a2_counters": r.a2_counters, "march_gbs": round(r.march_bytes / r.march_ns, 1),
                               "wall_ms_median": round(med(walls) / 1e6, 3)}})
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "locator_hbm_read_gbs": hbm_gbs, "by_setting": summary})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_l2_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
