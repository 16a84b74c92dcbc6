"""Markdown table of the per-kernel numbers of an `ncu --set full` report (one row per captured launch).
usage: python tools/ncu_step_summary.py report.ncu-rep > table.md"""
import csv
import subprocess
import sys

COLS = [("time µs", "gpu__time_duration.sum", 1.0, "{:.1f}"),
        ("DRAM rd MB", "dram__bytes_read.sum", 1.0, "{:.1f}"),
        ("DRAM wr MB", "dram__bytes_write.sum", 1.0, "{:.1f}"),
        ("warp-inst M", "smsp__inst_executed.sum", 1e-6, "{:.1f}"),
        ("issue active %", "smsp__issue_active.avg.pct_of_peak_sustained_active", 1.0, "{:.1f}"),
        ("warps active %", "sm__warps_active.avg.pct_of_peak_sustained_active", 1.0, "{:.1f}"),
        ("regs", "launch__registers_per_thread", 1.0, "{:.0f}"),
        ("alu pipe %", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", 1.0, "{:.1f}"),
        ("fma pipe %", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", 1.0, "{:.1f}"),
        ("xu pipe %", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", 1.0, "{:.1f}"),
        ("L1 wavefronts %", "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", 1.0, "{:.1f}")]
UNIT_SCALE = {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "nsecond": 1e-3, "second": 1e6,
              "byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}


PEAK = 3350.0     # GB/s, HBM3 bandwidth of the H100 SXM data sheet (not a measured figure)


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    ik, ig = hdr.index("Kernel Name"), hdr.index("Grid Size")
    print("| kernel | grid | " + " | ".join(c[0] for c in COLS) + " | DRAM GB/s | % of HBM peak |")
    print("|---|---|" + "---|" * (len(COLS) + 2))
    for r in rows[2:]:
        cells = []
        for _, key, scale, fmt in COLS:
            if key not in hdr:
                cells.append("—"); continue
            i = hdr.index(key)
            try:
                v = float(r[i].replace(",", ""))
            except ValueError:
                cells.append("—"); continue
            v *= UNIT_SCALE.get(units[i], 1.0) * scale
            cells.append(fmt.format(v))
        name = r[ik].split("(")[0].replace("void ", "").replace("borb::", "")
        try:                                   # achieved DRAM bandwidth of the launch against the measured HBM peak (MEASURED_PEAKS.json)
            gbs = (float(cells[1]) + float(cells[2])) * 1e6 / (float(cells[0]) * 1e-6) / 1e9
            cells += [f"{gbs:.0f}", f"{100 * gbs / PEAK:.1f}"]
        except ValueError:
            cells += ["—", "—"]
        print(f"| `{name}` | {r[ig]} | " + " | ".join(cells) + " |")


if __name__ == "__main__":
    main()
