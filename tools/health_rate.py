"""Spawn-to-exit time of the health check (one cro_check_health_uuid) against the six single helper forms with the same
options called one after another, on cuda:0.  JSON lines on stdout, and in <out-dir>/h100_<W>w_health.jsonl (W: the
card's power limit in watts).

The two arms alternate, --rounds times each, so both see the same clocks and the same host load.  Both scan the same
--scan-gib bytes (max_bytes), every other check runs with its defaults.  Per arm: spawn to exit (the sum of the six
helpers' for the singles), median, min and max, and each check's own leg time (its wall or CUDA-event time as the check
reports it), median; every call must come back clean.  The card's name, power limit and max SM clock come from a
read-only nvidia-smi query in the same run."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")


def med(xs):
    return sorted(xs)[len(xs) // 2]


def legs_ms(compute, precision, sram, l2, link, scan):
    """Each check's own time as it reports it: the legs' CUDA-event ns (compute, precision, SRAM, link), the call's
    wall ns (L2, scan)."""
    return {"compute": sum(L.ns for L in compute.leg) / 1e6, "precision": sum(L.ns for L in precision.leg) / 1e6,
            "sram": sum(L.ns for L in sram.leg) / 1e6, "l2": l2.wall_ns / 1e6, "link": sum(L.ns for L in link.leg) / 1e6,
            "scan": scan.wall_ns / 1e6}


def combined(uuid, scan_bytes):
    r, _, ns = cro.check_health_uuid(None, uuid, scan=dict(max_bytes=scan_bytes))
    assert r.status == cro.OK and r.ran == cro.HEALTH_ALL, (r.status, r.failed, r.errored, list(r.check_status))
    return ns, legs_ms(r.compute, r.precision, r.sram, r.l2, r.link, r.scan), [t / 1e6 for t in r.check_ns]


def singles(uuid, scan_bytes):
    c, _, _, c_ns = cro.probe_compute_uuid(None, uuid)
    p, _, _, p_ns = cro.probe_precision_uuid(None, uuid)
    s, _, _ = cro.probe_sram_uuid(None, uuid)
    l, _, _ = cro.probe_l2_uuid(None, uuid)
    k, _, k_ns = cro.probe_host_link_uuid(None, uuid)
    x, _ = cro.scan_hbm_uuid(None, uuid, max_bytes=scan_bytes)
    for name, r in (("compute", c), ("precision", p), ("sram", s), ("l2", l), ("link", k), ("scan", x)):
        assert r.status == cro.OK, (name, r.status)
    helpers = [c_ns, p_ns, s.helper_ns, l.helper_ns, k_ns, x.helper_ns]
    return sum(helpers), legs_ms(c, p, s, l, k, x), [h / 1e6 for h in helpers]


def stats(xs):
    return {"median": round(med(xs), 2), "min": round(min(xs), 2), "max": round(max(xs), 2)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--scan-gib", type=int, default=16)
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    scan_bytes = args.scan_gib << 30
    uuid = subprocess.run([os.path.join(os.path.dirname(cro.LIB_PATH), "croprobe-cli"), "csv", "gpu_uuid"], capture_output=True,
                          text=True, check=True).stdout.split()[0]
    combined(uuid, 1 << 30)                      # warm-up: page cache, driver, clocks
    arms = {"combined": [], "singles": []}
    for i in range(args.rounds):
        for arm, fn in (("combined", combined), ("singles", singles)) if i % 2 == 0 else (("singles", singles), ("combined", combined)):
            t0 = time.monotonic()
            ns, legs, per_check = fn(uuid, scan_bytes)
            arms[arm].append((ns / 1e6, legs, per_check, (time.monotonic() - t0) * 1e3))
            emit({"arm": arm, "round": i, "spawn_to_exit_ms": round(ns / 1e6, 2), "call_ms": round(arms[arm][-1][3], 2),
                  "per_check_ms": [round(t, 2) for t in per_check], "leg_ms": {k: round(v, 2) for k, v in legs.items()}})
    summary = {}
    for arm, runs in arms.items():
        summary[arm] = {"spawn_to_exit_ms": stats([r[0] for r in runs]),
                        "leg_ms": {k: round(med([r[1][k] for r in runs]), 2) for k in runs[0][1]}}
    saved = summary["singles"]["spawn_to_exit_ms"]["median"] - summary["combined"]["spawn_to_exit_ms"]["median"]
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "rounds": args.rounds, "scan_bytes": scan_bytes,
          "summary": summary, "saved_ms_median": round(saved, 2)})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_health.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
