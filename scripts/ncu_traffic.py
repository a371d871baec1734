#!/usr/bin/env python
"""Record the measured DRAM traffic of the dominant kernel for bench.py's `roofline.traffic`.

    python scripts/ncu_traffic.py <report.ncu-rep> --config 2 --chains 1048576 --sweeps-per-launch 50 [--note "..."]

Reads one `ncu --set full` capture of the SAME bench command, e.g.
`ncu --set full --clock-control none -k regex:amwg_jit_sweep -s 6 -c 1 -o prof_c2 python bench.py --steps 1 --warmup 1 --no-cpu`
(reading the report needs no GPU), and writes dram__bytes_read.sum + dram__bytes_write.sum of that launch into profiles/ncu_traffic.json,
keyed by config, together with the commit it was taken on. bench.py reads the file; nothing is hard-coded there."""
import argparse
import csv
import io
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("report")
    ap.add_argument("--config", type=int, required=True)
    ap.add_argument("--chains", type=int, required=True)
    ap.add_argument("--sweeps-per-launch", type=int, required=True)
    ap.add_argument("--note", default="")
    a = ap.parse_args()
    raw = subprocess.run(["ncu", "-i", a.report, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, vals = rows[0], rows[1], rows[-1]
    m = {h: (u, v) for h, u, v in zip(hdr, units, vals)}

    def num(key):
        u, v = m[key]
        x = float(v.replace(",", ""))
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}.get(u, 1)
        return x * scale
    rd, wr = num("dram__bytes_read.sum"), num("dram__bytes_write.sum")
    head = subprocess.run(["git", "-C", ROOT, "rev-parse", "--short", "HEAD"], capture_output=True, text=True).stdout.strip()
    entry = {"kernel": m.get("Kernel Name", ("", "?"))[1], "grid": m.get("Grid Size", ("", "?"))[1], "block": m.get("Block Size", ("", "?"))[1],
             "chains": a.chains, "sweeps_per_launch": a.sweeps_per_launch, "dram_bytes_read": rd, "dram_bytes_write": wr,
             "dram_bytes_per_launch": rd + wr, "duration_ns_under_ncu": m.get("gpu__time_duration.sum", ("", "?"))[1],
             "source": os.path.basename(a.report) + " @ " + head + (" -- " + a.note if a.note else "")}
    path = os.path.join(ROOT, "profiles", "ncu_traffic.json")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    data = {}
    if os.path.exists(path):
        with open(path) as f:
            data = json.load(f)
    data[f"config{a.config}"] = entry
    with open(path, "w") as f:
        json.dump(data, f, indent=1)
    print(json.dumps(entry, indent=1))


if __name__ == "__main__":
    main()
