#!/usr/bin/env python
"""Markdown table of a bench.py JSON line (headline + configs sub-records): python tools/bench_table.py bench_line.json
(a file holding the line bench.py printed)"""
import json
import sys


def row(name, r, head=False):
    k1, k2 = r["kernels"]["K1_picnn_fg"], r["kernels"]["K2_bundle_step"]
    cpu = r.get("cpu_baseline") or {}
    e2e = r["e2e"]
    lg = r.get("loop_graph") or {}
    return ("| %s%s | %.2f | %.3g | %.2f | %.3g | %.1f (%.1f %% / %.0f %%) | %.2f (%.1f %%) | %s | %s | %s |"
            % ("**" + name + "**" if head else name, " (headline)" if head else "", r["ms_per_step"], r["value"],
               e2e["ms_per_step"], e2e["value"], k1["achieved"], 100 * k1["frac"], 100 * k1["frac_of_3xtf32_ceiling"],
               k2["achieved"], 100 * k2["frac"],
               ("%.1f" % cpu["value"]) if cpu else "-", ("%.0f×" % (e2e["value"] / cpu["value"])) if cpu else "-",
               ("%.2f" % lg["ms_per_step"]) if lg else "-"))


def main():
    d = json.load(open(sys.argv[1]))
    print("| workload | device ms/step | device solves/s | e2e ms/step | e2e solves/s | K1 TFLOP/s (of bf16 peak / of 3×TF32 ceiling) "
          "| K2 FP64 TFLOP/s (of measured DMMA peak) | CPU port solves/s | e2e ÷ CPU | CUDA-graph ms/step |")
    print("|---|---:|---:|---:|---:|---|---|---:|---:|---:|")
    head = dict(d)
    head["ms_per_step"] = d["ms_per_step"]
    print(row(d["config"]["workload"].split(":")[0], head, True))
    for k, r in (d.get("configs") or {}).items():
        print(row(k, r))
    print()
    print("clocks", d.get("clocks"), "fp64 peak %.1f TFLOP/s" % d.get("fp64_mma_peak_tflops", 0), "steps", d["steps"], "warmup", d["warmup"])
    rc = (d.get("cpu_baseline") or {}).get("reference_cost")
    if rc:
        print("reference_cost %.3f solves/s (%s)" % (rc["value"], rc["sample"]))
    gd = (d.get("configs", {}).get("C3") or {}).get("gd_mode")
    if gd:
        print("C3 gd_mode", json.dumps(gd)[:600])


if __name__ == "__main__":
    main()
