#!/usr/bin/env python
"""Turn one `ncu --set full` report into a small JSON summary (DRAM bytes against the algorithmic bytes per launch).
    ncu -i prof.ncu-rep --page raw --csv > raw.csv     (no GPU needed)
    python tools/ncu_summary.py raw.csv --kernel verify_attn_mma_kernel --kv_len 124936 --rows 8 --heads 32 --head_dim 128 \
        --out summary.json
Units are read from the CSV's second header row and converted to bytes / microseconds."""
import argparse
import csv
import gzip
import json

UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "nsecond": 1e-3,
        "usecond": 1.0, "msecond": 1e3, "second": 1e6}
WANT = ["dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "lts__t_sector_hit_rate.pct", "sm__throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--kernel", required=True)
    ap.add_argument("--kv_len", type=int, required=True)
    ap.add_argument("--rows", type=int, required=True)
    ap.add_argument("--heads", type=int, required=True)
    ap.add_argument("--head_dim", type=int, default=128)
    ap.add_argument("--command", default="")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    op = gzip.open if args.csv.endswith(".gz") else open
    with op(args.csv, "rt", newline="") as f:
        rows = [r for r in csv.reader(f) if len(r) > 8]  # drops ncu's "==PROF==" log lines
    head = next(i for i, r in enumerate(rows) if r[0] == "ID")
    names, units = rows[head], rows[head + 1]
    col = {n: i for i, n in enumerate(names)}
    launches = []
    for r in rows[head + 2:]:
        if args.kernel not in r[col["Kernel Name"]]:
            continue
        rec = {"grid": r[col["Grid Size"]], "block": r[col["Block Size"]]}
        for w in WANT:
            if w in col:
                v = float(r[col[w]].replace(",", ""))
                rec[w] = v * UNIT.get(units[col[w]], 1.0)
        launches.append(rec)
    assert launches, f"no launch of {args.kernel} in {args.csv}"
    algo = args.kv_len * args.heads * args.head_dim * 2 * 2
    for rec in launches:
        rec["dram_bytes"] = rec["dram__bytes_read.sum"] + rec["dram__bytes_write.sum"]
        rec["traffic_over_algorithmic"] = rec["dram_bytes"] / algo
    out = dict(kernel=args.kernel, kv_len=args.kv_len, rows=args.rows, heads=args.heads, head_dim=args.head_dim, algorithmic_bytes=algo,
               units="bytes, microseconds, percent", command=args.command, launches=launches)
    json.dump(out, open(args.out, "w"), indent=1)
    print(json.dumps({k: out[k] for k in ("kernel", "kv_len", "algorithmic_bytes")}), [round(l["traffic_over_algorithmic"], 4) for l in launches])


if __name__ == "__main__":
    main()
