#!/usr/bin/env python3
"""ncu launch list (`--metrics gpu__time_duration.sum --csv --log-file x.csv`) -> per-kernel totals and shares, markdown.
    python tools/launch_summary.py validate_out/val_launches.csv [min_ms] > profiles/launches_summary.md
Only this library's kernels are listed (torch's synthetic-frame kernels are dropped); launches shorter than min_ms
(default 0: keep all) can be left out, e.g. the empty repair passes of the decoder."""
import csv
import sys


def main():
    path = sys.argv[1]
    min_ms = float(sys.argv[2]) if len(sys.argv) > 2 else 0.0
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    hdr, data = rows[0], rows[1:]
    ix = {h: i for i, h in enumerate(hdr)}
    per = {}
    for r in data:
        name = r[ix["Kernel Name"]]
        if not any(k in name for k in ("bc_encode_kernel", "bc_decode_kernel", "snappy_", "hap_")):     # (torch's kernels: at::native::...)
            continue
        short = name.split("(")[0].replace("hapb200::", "").replace("void ", "").strip()
        ms = float(r[ix["Metric Value"]]) * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(r[ix["Metric Unit"]], 1e-6)
        if ms < min_ms:
            continue
        n, t = per.get(short, (0, 0.0))
        per[short] = (n + 1, t + ms)
    total = sum(t for _, t in per.values()) or 1.0
    print("| kernel | launches | total ms | ms per launch | share |")
    print("|---|---|---|---|---|")
    for k, (n, t) in sorted(per.items(), key=lambda kv: -kv[1][1]):
        print(f"| `{k}` | {n} | {t:.3f} | {t / n:.3f} | {100 * t / total:.1f} % |")


if __name__ == "__main__":
    main()
