"""Rate of the fault locator's compare pass next to the LDG read sweep, on cuda:0 at S = 4 GiB.  One JSON line on stdout.

After one passing probe, 21 rounds alternate a pass-0 locate (both halves compared against the probe's pattern, 2 S
read) with one LDG read sweep (S read); each side's GB/s comes from the kernels' own %globaltimer windows and the
median is reported.  Then the wall time of a full locate with retest (two fills and two compare passes of both
halves, plus the closed forms), median of 5.  The GPU's name and power limit are read in the same run."""
import importlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")

S = 4 << 30
ROUNDS = 21


def med(xs):
    return sorted(xs)[len(xs) // 2]


def main() -> None:
    gpu, power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                capture_output=True, text=True, check=True).stdout.strip().split(", ")
    with cro.ProbeContext(sweep_bytes=S, devices=[0]) as ctx:
        assert ctx.probe_device(0).status == cro.OK
        for _ in range(3):      # warm-up of both kernels
            ctx.locate_faults(0, retest=False)
            ctx.hbm_read_checksum(0, cro.READ_LDG)
        scan, ldg = [], []
        for _ in range(ROUNDS):
            rep, words = ctx.locate_faults(0, retest=False)
            assert rep.verdict == cro.FAULTS_NONE and rep.complete == 1 and rep.pass_[0].halves == 3 and not words
            scan.append(rep.pass_[0].words_scanned * 8 / rep.pass_[0].scan_ns)
            r = ctx.hbm_read_checksum(0, cro.READ_LDG)
            ldg.append(r.bytes / r.timer_ns)
        walls = []
        for _ in range(5):
            t0 = time.perf_counter()
            rep, _ = ctx.locate_faults(0, retest=True)
            walls.append(time.perf_counter() - t0)
            assert rep.verdict == cro.FAULTS_NONE and rep.complete == 1
    scan_gbs, ldg_gbs = med(scan), med(ldg)
    print(json.dumps({"gpu": gpu, "power_limit": power, "sweep_bytes": S, "rounds": ROUNDS,
                      "pass0_scan_gbs_median": round(scan_gbs, 1), "ldg_read_gbs_median": round(ldg_gbs, 1),
                      "scan_over_ldg": round(scan_gbs / ldg_gbs, 3),
                      "locate_retest_wall_ms_median": round(med(walls) * 1e3, 2)}), flush=True)


if __name__ == "__main__":
    main()
