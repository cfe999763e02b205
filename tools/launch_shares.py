"""Per-kernel share of an ncu launch list (--metrics gpu__time_duration.sum --csv).
    python tools/launch_shares.py LAUNCHES.csv OUT.json"""
import csv, json, sys
rows = [r for r in csv.reader(open(sys.argv[1], errors="replace")) if len(r) > 5]
hdr = next(r for r in rows if "Kernel Name" in r)
ik, im, iv, iu = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
tot, per, n = 0.0, {}, {}
for r in rows:
    if r is hdr or r[im] != "gpu__time_duration.sum":
        continue
    v = float(r[iv].replace(",", "")) * {"ns": 1e-3, "us": 1.0, "ms": 1e3}.get(r[iu], 1.0)
    k = r[ik].split("(")[0].replace("void ", "").replace("srf::", "")
    per[k] = per.get(k, 0.0) + v; n[k] = n.get(k, 0) + 1; tot += v
out = {"total_us": tot, "kernels": {k: {"launches": n[k], "total_us": round(v, 1), "avg_us": round(v / n[k], 2), "share_pct": round(100 * v / tot, 2)}
                                    for k, v in sorted(per.items(), key=lambda kv: -kv[1])}}
json.dump(out, open(sys.argv[2], "w"), indent=1)
for k, d in list(out["kernels"].items())[:14]:
    print(f"{k[:60]:60s} {d['launches']:5d} {d['avg_us']:9.2f} us  {d['share_pct']:6.2f} %")
