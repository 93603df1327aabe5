"""Rates of the SM sparse probe's legs on cuda:0, next to PyTorch's own sparse (cuSPARSELt) and dense GEMMs in the same
run.  JSON lines on stdout, and in <out-dir>/h100_<W>w_sparse_rate.jsonl (W: the card's power limit in watts): one line
per grid point, then the PyTorch lines, then the summary line.

Rates are dense-equivalent: 2 M N K over the logical K, so a sparse GEMM that skips half the products and a dense one of
the same shape count the same operations.  Grid: for each leg and iteration count, the median over 21 calls of ops / ns
(ns: CUDA events around the launches of the leg, so the operand and metadata generation, the per-iteration fold and the
compare are inside it) and of the leg's time per call.  PyTorch: torch._cslt_sparse_mm on a 2:4-sparse 8192^3 product
in e4m3, int8, float16 and bfloat16, and the dense torch.matmul (float16, bfloat16), torch._int_mm (int8) and
torch._scaled_mm (e4m3) of the same shape; CUDA events, median of 21 after 3 warm-up calls.  A form this PyTorch build
cannot run is recorded with its error text instead of a rate.  PyTorch has no sparse TF32 or E5M2 GEMM to compare
with.  The card's name, power limit and max SM clock come from a read-only nvidia-smi query in the same run.  Last: 21
calls at the defaults, their wall time, host reference time and per-leg rates."""
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
ITERATIONS = [16, 256, 4096]
LEG_NAMES = ["s8", "e4m3", "e5m2", "bf16", "f16", "tf32"]
G = 8192


def med(xs):
    return sorted(xs)[len(xs) // 2]


def timed(fn):
    """Median CUDA-event time of fn() in ns, after 3 warm-up calls."""
    import torch
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
    return med(times)


def torch_gemms():
    import torch
    dev = torch.device("cuda", 0)
    mask = torch.tensor([1, 1, 0, 0], device=dev, dtype=torch.bool).repeat(G, G // 4)
    a = (torch.randint(1, 4, (G, G), device=dev) * mask).float()
    b = torch.randint(-3, 4, (G, G), device=dev).float()
    one = torch.ones((), device=dev)
    cases = {
        "f16": (torch.float16, lambda x, y: torch.matmul(x, y)),
        "bf16": (torch.bfloat16, lambda x, y: torch.matmul(x, y)),
        "int8": (torch.int8, lambda x, y: torch._int_mm(x, y)),
        "e4m3": (torch.float8_e4m3fn, lambda x, y: torch._scaled_mm(x, y, scale_a=one, scale_b=one, out_dtype=torch.bfloat16)),
    }
    out = []
    for name, (dt, dense) in cases.items():
        x = a.to(dt)
        yt = b.to(dt)                        # B^T, row-major: B is its column-major view
        for kind in ("sparse", "dense"):
            try:
                if kind == "sparse":
                    xc = torch._cslt_compress(x)
                    kw = dict(out_dtype=torch.bfloat16) if dt == torch.float8_e4m3fn else \
                        dict(out_dtype=torch.int32) if dt == torch.int8 else {}
                    ns = timed(lambda: torch._cslt_sparse_mm(xc, yt.t(), **kw))
                else:
                    ns = timed(lambda: dense(x, yt.t()))
                out.append({"torch": kind, "dtype": name, "shape": [G, G, G], "rate_median": int(2 * G ** 3 / ns)})
            except Exception as e:          # this build or card lacks the form: say so
                out.append({"torch": kind, "dtype": name, "shape": [G, G, G], "error": str(e).splitlines()[0][:200]})
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    best = {}
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0]) as ctx:
        ctx.probe_sparse(0, iterations=16)                          # warm-up: modules loaded, clocks up
        for it in ITERATIONS:
            for leg, name in enumerate(LEG_NAMES):
                rates, ns = [], []
                for _ in range(ROUNDS):
                    r, _s, _f = ctx.probe_sparse(0, legs=1 << leg, iterations=it)
                    L = r.leg[leg]
                    assert r.status == cro.OK, (name, it, L.mismatches, L.fold_mismatches)
                    rates.append(L.ops // L.ns)
                    ns.append(L.ns)
                emit({"leg": name, "iterations": it, "rate_median": med(rates), "leg_ns_median": med(ns)})
                best[name] = max(best.get(name, 0), med(rates))
        walls, host_ref, rates, leg_ns = [], [], {n: [] for n in LEG_NAMES}, {n: [] for n in LEG_NAMES}
        for _ in range(ROUNDS):
            t = time.perf_counter_ns()
            r, _s, _f = ctx.probe_sparse(0)
            walls.append(time.perf_counter_ns() - t)
            assert r.status == cro.OK
            host_ref.append(r.host_ref_ns)
            for leg, name in enumerate(LEG_NAMES):
                rates[name].append(r.leg[leg].ops // r.leg[leg].ns)
                leg_ns[name].append(r.leg[leg].ns)
        iterations, sm_count = r.leg[0].iterations, r.sm_count
    torch_lines = torch_gemms()
    for line in torch_lines:
        emit(line)
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "sm_count": sm_count, "rounds": ROUNDS,
          "rate_unit": "dense-equivalent GOP/s (s8) or GFLOP/s: 2 M N K over the logical K, per ns",
          "defaults": {"iterations": iterations}, "default_call_wall_ns_median": med(walls),
          "host_ref_ns_median": med(host_ref), "default_call_rate_median": {n: med(v) for n, v in rates.items()},
          "default_call_leg_ns_median": {n: med(v) for n, v in leg_ns.items()}, "best_grid_rate": best,
          "not_compared": ["tf32", "e5m2"]})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_sparse_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
