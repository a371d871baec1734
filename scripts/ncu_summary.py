#!/usr/bin/env python
"""Summarise an `ncu --set full` capture of the sweep kernel into a small markdown file.

    python scripts/ncu_summary.py prof.ncu-rep summary.md [--so path/to/libamwg_b200.so] [--warp-steps N]

Reads the report here (no GPU needed): raw metrics page + SASS source page. With --so the SASS page is split per device
function (the noinline functions are sub-symbols of the kernel) using `cuobjdump -elf`.
"""
import csv
import io
import re
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "launch__registers_per_thread", "launch__occupancy_limit_registers", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__issue_active.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__cycles_elapsed.avg.per_second",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sass__inst_executed_local_loads", "sass__inst_executed_local_stores"]
STALLS = "smsp__average_warps_issue_stalled_"


def run(cmd):
    return subprocess.run(cmd, capture_output=True, text=True).stdout


def main():
    rep, out = sys.argv[1], sys.argv[2]
    so = sys.argv[sys.argv.index("--so") + 1] if "--so" in sys.argv else None
    warp_steps = float(sys.argv[sys.argv.index("--warp-steps") + 1]) if "--warp-steps" in sys.argv else None
    raw = list(csv.reader(io.StringIO(run(["ncu", "-i", rep, "--page", "raw", "--csv"]))))
    hdr, units, vals = raw[0], raw[1], raw[-1]
    m = {h: (u, v) for h, u, v in zip(hdr, units, vals)}
    lines = [f"# ncu summary of `{rep.split('/')[-1]}`", "", f"kernel: `{m.get('Kernel Name', ('', '?'))[1]}`  grid {m.get('Grid Size', ('', '?'))[1]} block {m.get('Block Size', ('', '?'))[1]}", "",
             "| metric | value | unit |", "|---|---:|---|"]
    for k in KEYS:
        if k in m:
            lines.append(f"| {k} | {m[k][1]} | {m[k][0]} |")
    lines += ["", "Warp stall reasons (cycles per issued instruction):", "", "| reason | value |", "|---|---:|"]
    st = sorted(((h[len(STALLS):].replace("_per_issue_active.ratio", ""), float(v[1])) for h, v in m.items() if h.startswith(STALLS) and h.endswith("_per_issue_active.ratio")),
                key=lambda kv: -kv[1])
    for k, v in st[:9]:
        lines.append(f"| {k} | {v:.3f} |")
    src = list(csv.reader(io.StringIO(run(["ncu", "-i", rep, "--page", "source", "--csv"]))))
    h2, data = src[1], src[2:]
    iex, isamp, isrc = h2.index("Instructions Executed"), h2.index("# Samples"), h2.index("Source")
    ex = [int(r[iex] or 0) for r in data]
    sm = [int(r[isamp] or 0) for r in data]
    lines += ["", f"SASS: {len(data)} instructions in the kernel image, {sum(1 for e in ex if e)} executed at least once, {sum(ex)} warp-instructions executed."]
    ops = {}
    for r, e in zip(data, ex):
        mm = re.match(r"\s*(@!?U?P\d+\s+)?([A-Z0-9_]+)", r[isrc])
        if mm:
            ops[mm.group(2)] = ops.get(mm.group(2), 0) + e
    top = sorted(ops.items(), key=lambda kv: -kv[1])[:10]
    lines += ["", "Executed instruction mix: " + ", ".join(f"{k} {v / max(sum(ex), 1):.1%}" for k, v in top)]
    if so:
        elf = run(["cuobjdump", "-elf", so])
        kern = m.get("Kernel Name", ("", ""))[1].split("(")[0].split("::")[-1].replace("void ", "").strip()
        targ = ""
        if "<" in kern:                                   # template instantiation, e.g. amwg_sweep_kernel<0> -> ...kernelILb0EE
            kern, arg = kern.split("<", 1)
            targ = "ILb" + arg.rstrip(">").strip() + "E"
        funcs = []
        for ln in elf.splitlines():
            mm = re.match(r"\s+0x[0-9a-f]+\s+(0x[0-9a-f]+)\s+(0x[0-9a-f]+)\s+0x2\s+\S+\s+\S+\s+\$_ZN4amwg" + str(len(kern)) + kern + targ + r"E[^$]*\$(\S+)", ln)
            if mm:
                funcs.append((int(mm.group(1), 16) // 16, int(mm.group(2), 16) // 16, mm.group(3)))
        funcs.sort()
        if funcs:
            regions = [(0, funcs[0][0], "kernel body (sweep loop, steppers, rnorm)")] + [(a, a + n, name) for a, n, name in funcs]
            lines += ["", "Per device function (share of executed warp-instructions / of stall samples" + (", instructions per warp-step" if warp_steps else "") + "):", "",
                      "| function | SASS instrs | executed share | sample share |" + (" instrs/warp-step |" if warp_steps else ""), "|---|---:|---:|---:|" + ("---:|" if warp_steps else "")]
            for a, b, name in regions:
                e, s = sum(ex[a:b]), sum(sm[a:b])
                if e == 0 and s == 0:
                    continue
                name = re.sub(r"^_ZN4amwg\d+", "", name)
                name = re.sub(r"E[A-Za-z0-9_]*$", "", name) if name.startswith(("run_", "plate_", "philox", "js_", "cold")) else name
                row = f"| {name} | {b - a} | {e / max(sum(ex), 1):.3f} | {s / max(sum(sm), 1):.3f} |"
                if warp_steps:
                    row += f" {e / warp_steps:.0f} |"
                lines.append(row)
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
