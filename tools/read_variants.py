"""Where the AUTO read choice should switch, and a cross-check of the kernels' rates.  JSON lines on stdout.

1. Whole probes (graph replay) with the read variant forced, S = 64 MiB .. 4 GiB, median of 21 after 5 warm-up probes:
   probe time, and the best read / copy / fill sweep of those probes as GB/s (the kernels' own %globaltimer windows).
2. The same kinds of traffic through PyTorch's own kernels on a 4 GiB int64 tensor, CUDA events around 20 launches
   after 3 warm-up ones: fill_ (S written), copy_ (2*S moved), sum (S read).  An independent figure for the same GPU,
   so that a rate from the probe's kernels can be compared with something that does not share their timing code.
The first line names the GPU, its power limit and its maximum SM clock."""
import importlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
cro = importlib.import_module("composable-resource-operator_b200")
smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": smi}), flush=True)


def med(xs):
    return sorted(xs)[len(xs) // 2]


for mib in (64, 128, 256, 512, 1024, 2048, 4096):
    S = mib << 20
    for v in (cro.READ_LDG, cro.READ_TMA, cro.READ_LDG256):
        with cro.ProbeContext(sweep_bytes=S, devices=[0], read_variant=v) as c:
            for _ in range(5):
                c.probe_device(0)
            rs = [c.probe_device(0) for _ in range(21)]
            assert all(r.status == 0 and r.copy_verified == 5 and r.read_variant == v for r in rs)
            print(json.dumps({"mib": mib, "read_variant": v, "probe_us_median": round(med([r.total_ns for r in rs]) / 1e3, 1),
                              "read_gbs_best": round(S / min(r.read_best_ns for r in rs), 1),
                              "copy_gbs_best": round(2 * S / min(r.copy_best_ns for r in rs), 1),
                              "fill_gbs_best": round(S / min(r.fill_ns for r in rs), 1)}), flush=True)

import torch  # noqa: E402  (after every probe context is closed)

S = 4 << 30
x = torch.empty(S // 8, dtype=torch.int64, device="cuda")
y = torch.empty_like(x)
for name, moved, fn in (("torch fill_", S, lambda: x.fill_(7)), ("torch copy_", 2 * S, lambda: y.copy_(x)),
                        ("torch sum", S, lambda: x.sum())):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        fn()
    b.record()
    b.synchronize()
    print(json.dumps({"kernel": name, "bytes": moved, "gbs_mean_of_20": round(20 * moved / (a.elapsed_time(b) * 1e6), 1)}), flush=True)
