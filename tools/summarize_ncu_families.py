"""<dir>/*.raw.csv (ncu --set full, `--page raw --csv`, one capture per kernel family) -> one markdown table.

    python tools/summarize_ncu_families.py <ncu report dir> > ncu_families.md

One row per captured launch: grid, registers, duration, DRAM bytes read / written, achieved DRAM GB/s and its fraction of
the measured HBM peak (MEASURED_PEAKS.json), ncu's DRAM- and SM-throughput percentages and the L2 hit rate."""
import csv
import glob
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def to_bytes(v: str, unit: str) -> float:
    x = float(v.replace(",", ""))
    return x * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)


def to_us(v: str, unit: str) -> float:
    x = float(v.replace(",", ""))
    return x * {"ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6}.get(unit, 1)


def main():
    d = sys.argv[1]
    peak = 6571.2
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            peak = float(json.load(f)["hbm_gbs"])
    except Exception:
        pass
    print("| capture | kernel | grid x block | regs | duration (us) | dram read | dram written | DRAM GB/s | of measured peak "
          f"({peak:.1f}) | dram % | sm % | L2 hit % |")
    print("|---|---|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|")
    for path in sorted(glob.glob(os.path.join(d, "*.raw.csv"))):
        cap = os.path.basename(path)[4:-8]
        rows = list(csv.reader(open(path)))
        if len(rows) < 3:
            continue
        hdr, units = rows[0], rows[1]
        col = {n: i for i, n in enumerate(hdr)}

        def get(r, name):
            return r[col[name]], units[col[name]]

        for r in rows[2:]:
            name = re.sub(r"^void (ssdk::)?", "", r[col["Kernel Name"]])
            name = re.sub(r"\(.*$", "", name)
            dur = to_us(*get(r, "gpu__time_duration.sum"))
            rd, wr = to_bytes(*get(r, "dram__bytes_read.sum")), to_bytes(*get(r, "dram__bytes_write.sum"))
            gbs = (rd + wr) / (dur * 1e-6) / 1e9 if dur > 0 else 0.0
            grid = r[col["Grid Size"]].replace(" ", "") + "x" + r[col["Block Size"]].replace(" ", "")

            def pct(metric):
                return f"{float(r[col[metric]].replace(',', '')):.1f}" if metric in col and r[col[metric]] not in ("", "n/a") else "-"

            print(f"| {cap} | `{name}` | {grid} | {r[col['launch__registers_per_thread']]} | {dur:.2f} | {rd / 1e6:.3f} MB | "
                  f"{wr / 1e6:.3f} MB | {gbs:.0f} | {gbs / peak:.3f} | {pct('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed')} | "
                  f"{pct('sm__throughput.avg.pct_of_peak_sustained_elapsed')} | {pct('lts__t_sector_hit_rate.pct')} |")


if __name__ == "__main__":
    main()
