"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list into per-kernel means and shares.

usage: python scripts/summarize_launches.py launches.csv > launch_shares.json
The bench command under ncu runs the update several times (warm-up + timed steps); every kernel of the update appears
once per step, so mean duration per kernel name x launches per step = the step's kernel time."""
import csv
import json
import re
import sys
from collections import OrderedDict


# kernels of the public-API calls that BUILD the workload (propagate / augmentState / prune), not of the timed update
SETUP_KERNELS = {"k_propagate", "k_augment", "k_gather"}


def main(path):
    rows = []
    with open(path, newline="") as f:
        lines = [l for l in f if not l.startswith("==")]
    rd = csv.DictReader(lines)
    for r in rd:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        name = r["Kernel Name"]
        m = re.search(r"(k_[a-z_0-9]+)", name)
        if not m or m.group(1) in SETUP_KERNELS:
            continue
        val = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "ns")
        us = val / 1e3 if unit in ("ns", "nsecond") else (val if unit in ("us", "usecond") else val * 1e3)
        rows.append((m.group(1), us))
    per = OrderedDict()
    for k, us in rows:
        per.setdefault(k, []).append(us)
    steps = min(len(v) for v in per.values())
    kernels = [{"kernel": k, "launches": len(v), "launches_per_step": len(v) / steps, "mean_us": sum(v) / len(v)} for k, v in per.items()]
    total = sum(k["mean_us"] * k["launches_per_step"] for k in kernels)
    for k in kernels:
        k["share_pct"] = 100.0 * k["mean_us"] * k["launches_per_step"] / total
    kernels.sort(key=lambda k: -k["share_pct"])
    json.dump({"per_step_us": total, "steps_seen": steps, "kernels": kernels}, sys.stdout, indent=1)
    print()


if __name__ == "__main__":
    main(sys.argv[1])
