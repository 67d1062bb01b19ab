#!/usr/bin/env python
"""Regenerates profiles/traffic.json (roofline.traffic of bench.py) from an ncu capture instead of by hand.

    # on the GPU box (EPP_DEV_CHUNKS=1: every launch covers the whole batch, like the synchronous pass whose CUDA-event
    # time bench.py divides the bytes by)
    EPP_DEV_CHUNKS=1 ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none \\
        -k regex:'k_hash_fused|k_match_pick_sparse' -s 6 -c 4 --csv --log-file traffic.csv \\
        python bench.py --no-e2e --no-cpu --no-index-write --no-full-index --steps 2 --warmup 3
    # here
    python tools/ncu_traffic.py traffic.csv config3

Per kernel the capture's LAST launch is kept (steady state); traffic = dram read + write bytes of that launch."""
import csv
import json
import os
import sys


def main(path, workload):
    rows = [r for r in csv.reader(open(path)) if r and not r[0].startswith("==")]
    hdr = rows[0]
    ix = {h: i for i, h in enumerate(hdr)}
    per = {}
    for r in rows[1:]:
        if len(r) < len(hdr):
            continue
        name = r[ix["Kernel Name"]].split("(")[0].split("<")[0].replace("void ", "").split("::")[-1]
        metric, unit, val = r[ix["Metric Name"]], r[ix["Metric Unit"]], float(r[ix["Metric Value"]].replace(",", ""))
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1, "us": 1e3, "ms": 1e6}.get(unit, 1)
        per.setdefault(name, {}).setdefault(r[ix["ID"]], {})[metric] = val * scale
    out_path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "traffic.json")
    out = json.load(open(out_path)) if os.path.exists(out_path) else {}
    for name, launches in per.items():
        last = launches[sorted(launches, key=int)[-1]]
        traffic = int(last.get("dram__bytes_read.sum", 0) + last.get("dram__bytes_write.sum", 0))
        out[f"{workload}:{name}"] = traffic
        print(f"{workload}:{name}: read {last.get('dram__bytes_read.sum', 0) / 1e6:.1f} MB, written "
              f"{last.get('dram__bytes_write.sum', 0) / 1e6:.1f} MB, {last.get('gpu__time_duration.sum', 0) / 1e3:.1f} us")
    out["_how"] = "tools/ncu_traffic.py from an ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum capture of bench.py (see the script header)"
    json.dump(out, open(out_path, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "config3")
