"""Runs BASELINE.json configs 3, 4 and 5 on the box's GPUs (single process, as a Go operator would) and prints
one JSON object per config.  Config 2 is bench.py; config 1 is `bench.py --impl reference`.

  config 3  8xH100 full-box compose: cro_probe_all (concurrent probes + NVLink rounds + one NCCL all-gather)
  config 4  reconcile storm: 1000 synthetic ComposabilityRequests over the box's GPUs, warm probe contexts
  config 5  attach/detach churn: 100 cycles x 4-GPU compose / decompose, probe each attach

Usage: python tools/run_configs.py [--sweep-gib 4] [--storm 1000] [--cycles 100] [--configs 3,4,5]
"""
import argparse
import importlib
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import __graft_entry__ as g  # noqa: E402

g.build()
cro = importlib.import_module("composable-resource-operator_b200")

ap = argparse.ArgumentParser()
ap.add_argument("--sweep-gib", type=float, default=4.0)
ap.add_argument("--storm", type=int, default=1000)
ap.add_argument("--cycles", type=int, default=100)
ap.add_argument("--configs", default="3,4,5")
ap.add_argument("--cpu-compare", action="store_true", help="also run storm/churn with the probe off (reference-strength check)")
args = ap.parse_args()
S = int(args.sweep_gib * (1 << 30))
which = set(args.configs.split(","))


# the three legs live in bench.py (the driver runs them there for N > 1); this script runs them alone
import bench  # noqa: E402
import oracle  # noqa: E402


def config3(ctx):
    return dict(bench.fullbox_leg(cro, ctx, S, 5, 1, oracle.COracle()), config=3)


def storm(ctx, n_req, probe):
    return bench.storm_leg(cro, ctx, n_req, probe)


def churn(ctx, cycles, probe):
    return bench.churn_leg(cro, ctx, cycles, probe)


t0 = time.perf_counter()
ctx = cro.ProbeContext(sweep_bytes=S)
init_s = time.perf_counter() - t0
print(json.dumps({"init": {"devices": ctx.device_count(), "cold_init_s": round(init_s, 3), "sweep_bytes": S}}), flush=True)
if "3" in which:
    print(json.dumps(config3(ctx)), flush=True)
if "4" in which:
    print(json.dumps(storm(ctx, args.storm, True)), flush=True)
    if args.cpu_compare:
        print(json.dumps(storm(ctx, args.storm, False)), flush=True)
if "5" in which:
    print(json.dumps(churn(ctx, args.cycles, True)), flush=True)
    if args.cpu_compare:
        print(json.dumps(churn(ctx, args.cycles, False)), flush=True)
ctx.close()
