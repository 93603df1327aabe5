"""Rates of the host link probe's legs on cuda:0 at L = 1 GiB.  JSON lines on stdout, and with --out in that file too:
one line per grid point, then the summary line.

First the grid of the SM legs: for each CTA count, 3 calls, median MB/s of the SM h2d, d2h and duplex legs (events).
Then 21 calls at the default grid, median per leg.  The GPU's name and power limit come from nvidia-smi in the same
run, and the trained link (current and max speed and width, sampled during the copy-engine duplex leg) from the
result itself.

--helper: instead, the helper form (cro_probe_host_link_uuid) against the in-process form at L = 256 MiB, the helper's
default: HELPER_ROUNDS calls of each, alternating, in one context over cuda:0.  One line: the median, least and largest
spawn-to-exit time of the helper, and per leg the median MB/s inside the helper and in process."""
import argparse
import importlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")

L = 1 << 30
ROUNDS = 21
GRIDS = [1, 2, 4, 8, 16, 32, 66, 132]
HELPER_L = 256 << 20
HELPER_ROUNDS = 9
LEGS = ["ce_d2h", "sm_h2d", "ce_h2d", "sm_d2h", "sm_duplex_h2d", "sm_duplex_d2h", "ce_duplex_h2d", "ce_duplex_d2h"]


def med(xs):
    return sorted(xs)[len(xs) // 2]


def mbps(nbytes, ns):
    return nbytes * 1000 // ns if ns else 0


def speed(t):
    return "unknown" if t == 0 else "%d.%dGT/s" % (t // 10, t % 10)


def helper_rates(gpu: str, power: str) -> dict:
    with cro.ProbeContext(sweep_bytes=HELPER_L, devices=[0]) as ctx:
        uuid = ctx.own_devices()[0].gpu_uuid.decode()
        ctx.probe_host_link(0, bytes=HELPER_L)                      # warm-up: host buffers pinned, link trained up
        cro.probe_host_link_uuid(ctx, uuid, bytes=HELPER_L)
        inproc, helper, spawn = [], [], []
        for _ in range(HELPER_ROUNDS):
            r, _f = ctx.probe_host_link(0, bytes=HELPER_L)
            assert r.status == cro.OK, r.first_fail
            inproc.append(r)
            r, _f, ns = cro.probe_host_link_uuid(ctx, uuid, bytes=HELPER_L)
            assert r.status == cro.OK, r.first_fail
            helper.append(r)
            spawn.append(ns)
    out = {"gpu": gpu, "power_limit": power, "probe": "host_link", "bytes": HELPER_L, "rounds": HELPER_ROUNDS,
           "helper_ns_median": med(spawn), "helper_ns_min": min(spawn), "helper_ns_max": max(spawn),
           "legs_ns_median": {"helper": med([sum(g.ns for g in r.leg) for r in helper]),
                              "in_process": med([sum(g.ns for g in r.leg) for r in inproc])}}
    for i, name in enumerate(LEGS):
        out[name + "_mbps_median"] = {"helper": med([mbps(r.leg[i].bytes, r.leg[i].ns) for r in helper]),
                                      "in_process": med([mbps(r.leg[i].bytes, r.leg[i].ns) for r in inproc])}
    out["latency_ns_median"] = {"helper": med([r.chase_ns // r.chase_hops for r in helper]),
                                "in_process": med([r.chase_ns // r.chase_hops for r in inproc])}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--helper", action="store_true", help="the helper form against the in-process form")
    args = ap.parse_args()
    lines = []

    def emit(line):
        print(line, flush=True)
        lines.append(line)

    gpu, power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                capture_output=True, text=True, check=True).stdout.strip().split(", ")
    if args.helper:
        emit(json.dumps(helper_rates(gpu, power)))
        if args.out:
            with open(args.out, "a") as f:
                f.write("\n".join(lines) + "\n")
        return
    with cro.ProbeContext(sweep_bytes=L, devices=[0]) as ctx:
        assert ctx.probe_device(0).status == cro.OK
        for _ in range(2):       # warm-up: host buffers allocated and pinned, link trained up
            ctx.probe_host_link(0, bytes=L)
        for g in GRIDS:
            rows = []
            for _ in range(3):
                r, _f = ctx.probe_host_link(0, bytes=L, ctas=g)
                assert r.status == cro.OK, r.first_fail
                rows.append(r)
            emit(json.dumps({"ctas": g,
                              "sm_h2d_mbps": med([mbps(L, r.leg[1].ns) for r in rows]),
                              "sm_d2h_mbps": med([mbps(L, r.leg[3].ns) for r in rows]),
                              "sm_duplex_mbps": med([mbps(2 * L, r.leg[4].ns) for r in rows])}))
        rows = []
        for _ in range(ROUNDS):
            r, _f = ctx.probe_host_link(0, bytes=L)
            assert r.status == cro.OK, r.first_fail
            rows.append(r)
    last = rows[-1]
    g0 = last.path.hop[0]
    out = {"gpu": gpu, "power_limit": power, "bytes": L, "rounds": ROUNDS,
           "link": "%s x%d / %s x%d" % (speed(g0.cur_speed), g0.cur_width, speed(g0.max_speed), g0.max_width),
           "path_hops": last.path.n_hops, "degraded": last.degraded, "dev_numa": last.dev_numa,
           "host_numa": list(last.host_numa), "no_nvml": last.no_nvml,
           "replays": sum(r.replays_after - r.replays_before for r in rows) if not last.no_nvml else None}
    for i, name in enumerate(LEGS):
        out[name + "_mbps_median"] = med([mbps(r.leg[i].bytes, r.leg[i].ns) for r in rows])
    out["sm_duplex_mbps_median"] = med([mbps(2 * L, r.leg[4].ns) for r in rows])
    out["ce_duplex_mbps_median"] = med([mbps(2 * L, r.ce_duplex_span_ns) for r in rows])
    out["latency_ns_median"] = med([r.chase_ns // r.chase_hops for r in rows])
    out["path_cur"] = [(last.path.hop[i].bdf.decode(), last.path.hop[i].cur_speed, last.path.hop[i].cur_width,
                        last.path.hop[i].max_speed, last.path.hop[i].max_width) for i in range(last.path.n_hops)]
    emit(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
