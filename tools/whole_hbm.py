"""One probe over (nearly) the whole HBM of an H100: S = 36 GiB per half, a 72 GiB region of the 80 GB part
(falls back to 34 / 32 / 28 GiB if the allocation is refused).  Every sweep against the C oracle's closed form — word
indices run past 2^32.  JSON line on stdout."""
import importlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import __graft_entry__ as g

g.build()
cro = importlib.import_module("composable-resource-operator_b200")
import oracle  # noqa: E402  (the checker)

co = oracle.COracle()
for gib in (36, 34, 32, 28):
    S = gib << 30
    try:
        ctx = cro.ProbeContext(sweep_bytes=S, devices=[0])
    except cro.ProbeError as e:
        print(json.dumps({"sweep_gib": gib, "refused": str(e)}), flush=True)
        continue
    with ctx as c:
        probes = [c.probe_device(0) for _ in range(3)]
        r = probes[0]
        t0 = time.time()
        want = co.checksum(r.seed, 0, S // 8, threads=os.cpu_count() or 1)
        oracle_s = time.time() - t0
        ok = all(p.status == 0 and p.copy_verified == 5 for p in probes) and r.checksum == r.copy_checksum == r.expect == want
        best = min(p.total_ns for p in probes)
        print(json.dumps({"sweep_gib": gib, "region_gib": 2 * gib, "parity_ok": bool(ok), "probe_ms": round(best / 1e6, 2),
                          "probe_effective_gbs": round(16 * S / best, 1), "read_best_gbs": round(S / r.read_best_ns, 1),
                          "copy_best_gbs": round(2 * S / r.copy_best_ns, 1), "fill_gbs": round(S / r.fill_ns, 1),
                          "oracle_seconds_on_host": round(oracle_s, 1), "host_threads": os.cpu_count()}), flush=True)
        sys.exit(0 if ok else 3)
sys.exit(4)
