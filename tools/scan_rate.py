"""Rates and wall-time split of the whole-HBM scan on cuda:0.  JSON lines on stdout, and in
<out-dir>/h100_<W>w_scan_rate.jsonl (W: the card's power limit in watts): one line per size and form, then the summary.

Per size (--sizes-gib, 1, 4 and 16 GiB by default; the whole free memory but the 1 GiB reserve only with --all): the
in-process scan (cro_scan_hbm), median over --rounds calls of each element's GB/s (bytes / ns, ns from the CUDA events around the
element), and of the wall time split into allocation (cudaMalloc + cudaFree of the chunks), elements, NVML reads and the
rest; then the same scan through the helper process (cro_scan_hbm_uuid), whose extra time over the scan itself is the
helper's start (exec, cuInit, context, NVML init), the transfer of the report and its exit.  The card's name, power
limit and max SM clock come from a read-only nvidia-smi query in the same run."""
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


def split(rep):
    el = sum(rep.element_ns)
    return {"covered_bytes": rep.covered_bytes, "chunks": rep.n_chunks,
            "element_gbs": [round(rep.covered_bytes / ns, 1) if ns else 0 for ns in rep.element_ns],
            "alloc_ns": rep.alloc_ns, "elements_ns": el, "nvml_ns": rep.nvml_ns,
            "other_ns": rep.wall_ns - rep.alloc_ns - el - rep.nvml_ns, "wall_ns": rep.wall_ns}


def medians(splits):
    out = {k: med([s[k] for s in splits]) for k in splits[0] if k != "element_gbs"}
    out["element_gbs"] = [med([s["element_gbs"][e] for s in splits]) for e in range(4)]
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes-gib", default="1,4,16", help="comma-separated scan sizes in GiB")
    ap.add_argument("--all", action="store_true", help="also scan the whole free memory (all of it but the reserve)")
    args = ap.parse_args()
    lines = []

    def emit(obj):
        line = json.dumps(obj)
        print(line, flush=True)
        lines.append(line)

    gpu, power, clock = subprocess.run(
        ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True, check=True).stdout.strip().split(", ")
    sizes = [int(g) << 30 for g in args.sizes_gib.split(",")] + ([0] if args.all else [])
    summary = {}
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as ctx:
        uuid = ctx.own_devices()[0].gpu_uuid.decode()
        ctx.scan_hbm(0, max_bytes=256 << 20)                        # warm-up: modules loaded, clocks up
        for size in sizes:
            splits = []
            for _ in range(args.rounds):
                rep, _w = ctx.scan_hbm(0, max_bytes=size)
                assert rep.status == cro.OK, (size, rep.status, rep.pass_[0].mismatches, rep.pass_[1].mismatches)
                splits.append(split(rep))
            m = medians(splits)
            emit({"form": "in-process", "max_bytes": size, "rounds": args.rounds, **m})
            helper = []
            for _ in range(max(1, args.rounds // 2)):
                rep, _w = cro.scan_hbm_uuid(None, uuid, max_bytes=size)
                assert rep.status == cro.OK, (size, rep.status)
                s = split(rep)
                s["helper_ns"] = rep.helper_ns
                s["helper_start_and_transfer_ns"] = rep.helper_ns - rep.wall_ns
                helper.append(s)
            h = medians(helper)
            emit({"form": "helper", "max_bytes": size, "rounds": len(helper), **h})
            summary[str(size >> 30) if size else "all"] = {"in_process_wall_ns": m["wall_ns"], "helper_ns": h["helper_ns"],
                                                           "element_gbs": m["element_gbs"]}
    emit({"gpu": gpu, "power_limit": power, "clocks_max_sm": clock, "summary_by_gib": summary})
    watts = int(float(power.split()[0]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "h100_%dw_scan_rate.jsonl" % watts), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
