#!/usr/bin/env python
"""Summarise an Nsight Compute report (run here, no GPU needed):  key raw metrics + stall-reason histogram + hottest SASS.

    python scripts/summarize_ncu.py prof.ncu-rep summary.md [title]
"""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "sm__cycles_elapsed.avg.per_second"]


def page(rep, name):
    out = subprocess.run(["ncu", "-i", rep, "--page", name, "--csv"], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    rep, dst = sys.argv[1], sys.argv[2]
    title = sys.argv[3] if len(sys.argv) > 3 else rep
    raw = page(rep, "raw")
    hdr, units = raw[0], raw[1]
    lines = [f"# {title}", "", f"source report: `{rep}` (ncu --set full --clock-control none --import-source on)", ""]
    for r in raw[2:]:
        d = dict(zip(hdr, r))
        lines += [f"## {d.get('Kernel Name', '?')[:110]}", "", "| metric | value | unit |", "|---|---|---|"]
        for k in KEYS:
            if k in d and d[k] != "":
                lines.append(f"| {k} | {d[k]} | {units[hdr.index(k)]} |")
        try:
            rd = float(d["dram__bytes_read.sum"])
            wr = float(d["dram__bytes_write.sum"])
            ur, uw = units[hdr.index("dram__bytes_read.sum")], units[hdr.index("dram__bytes_write.sum")]
            scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
            tot = rd * scale[ur] + wr * scale[uw]
            t = float(d["gpu__time_duration.sum"]) * {"ns": 1e-9, "us": 1e-6, "ms": 1e-3}[units[hdr.index("gpu__time_duration.sum")]]
            lines.append(f"| dram traffic per launch (read+write) | {tot / 1e9:.4f} | GB |")
            lines.append(f"| dram GB/s under ncu (cold, serialised) | {tot / t / 1e9:.1f} | GB/s |")
        except Exception:
            pass
        tot_s = float(d.get("smsp__pcsamp_sample_count", 0) or 0)
        stalls = sorted(((float(d[k]), k) for k in hdr if "pcsamp_warps_issue_stalled" in k and "not_issued" not in k
                         and d[k] not in ("", "0")), reverse=True)
        if tot_s:
            lines += ["", "| warp stall reason (pc sampling) | samples | share |", "|---|---|---|"]
            for v, k in stalls[:10]:
                lines.append(f"| {k.replace('smsp__pcsamp_warps_issue_stalled_', '')} | {v:.0f} | {100 * v / tot_s:.1f}% |")
        lines.append("")
    src = page(rep, "source")
    if len(src) > 2:
        h = src[1]
        try:
            ia, isamp, iex = h.index("Source"), h.index("# Samples"), h.index("Instructions Executed")
            rows = []
            for r in src[2:]:
                if len(r) < len(h):
                    continue
                try:
                    rows.append((int(r[isamp] or 0), int(r[iex] or 0), r[ia]))
                except ValueError:
                    pass
            tot = sum(x[0] for x in rows) or 1
            agg = {}
            for s_, e_, text in rows:
                op = text.split()[1] if text.startswith("@") else text.split()[0]
                a = agg.setdefault(op, [0, 0])
                a[0] += s_
                a[1] += e_
            lines += ["## hottest SASS opcodes (first kernel in the report)", "", "| opcode | samples | share | executed |",
                      "|---|---|---|---|"]
            for op, (s_, e_) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:14]:
                lines.append(f"| {op} | {s_} | {100 * s_ / tot:.1f}% | {e_} |")
        except ValueError:
            pass
    open(dst, "w").write("\n".join(lines) + "\n")
    print("wrote", dst)


if __name__ == "__main__":
    main()
