"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list into a markdown table."""
import collections
import csv
import re
import sys

src, dst, title = sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else "launch list"
with open(src) as f:
    lines = [l for l in f if not l.startswith("==")]
agg = collections.defaultdict(lambda: [0, 0.0])
seq = []
for row in csv.DictReader(lines):
    name = re.sub(r"\(.*", "", row["Kernel Name"]).replace("void ", "").replace("ssdk::", "")
    v = float(row["Metric Value"].replace(",", ""))
    unit = row["Metric Unit"]
    v = v / 1000 if unit in ("nsecond", "ns") else (v * 1000 if unit in ("msecond", "ms") else v)
    agg[name][0] += 1
    agg[name][1] += v
    seq.append((name, v))
tot = sum(v for _, v in seq)
with open(dst, "w") as out:
    out.write(f"# {title}\n\n")
    out.write("`ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off` over ONE speculative step "
              "(`tools/profile_step.py`): per-launch times are cold-cache and serialised (ncu flushes caches and breaks PDL overlap), "
              "so compare SHARES, not absolutes.\n\n")
    out.write(f"launches in the step: **{len(seq)}**, sum of serialised kernel time: **{tot / 1000:.2f} ms**\n\n")
    out.write("| kernel | launches | total us | avg us | share |\n|---|---:|---:|---:|---:|\n")
    for k, (n, t) in sorted(agg.items(), key=lambda x: -x[1][1]):
        out.write(f"| `{k}` | {n} | {t:.1f} | {t / n:.2f} | {t / tot * 100:.1f}% |\n")
print("wrote", dst)
