"""Per-kernel summary of an ncu launch list (csv with gpu__time_duration.sum and, optionally, dram__bytes_read/write.sum):
launches, total ms, share, mean us, DRAM GB/s.   python tools/summarize_launches.py <ncu launch list .csv> [skip_first_n]"""
import csv, re, sys
path = sys.argv[1]
skip = int(sys.argv[2]) if len(sys.argv) > 2 else 0
rows = list(csv.reader(l for l in open(path) if l.startswith('"')))
hdr = rows[0]
ix = {h: i for i, h in enumerate(hdr)}
scale_t = {"ns": 1e-3, "nsecond": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "second": 1e6}
scale_b = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "B": 1.0, "KB": 1e3, "MB": 1e6, "GB": 1e9}
per = {}
for r in rows[1:]:
    kid = int(r[ix["ID"]])
    if kid < skip:
        continue
    name = re.sub(r"\(.*", "", r[ix["Kernel Name"]])
    name = re.sub(r"^void ", "", name)
    d = per.setdefault((kid, name), {})
    v = float(r[ix["Metric Value"]].replace(",", ""))
    m, u = r[ix["Metric Name"]], r[ix["Metric Unit"]]
    if m == "gpu__time_duration.sum": d["us"] = v * scale_t.get(u, 1.0)
    elif m == "dram__bytes_read.sum": d["rd"] = v * scale_b.get(u, 1.0)
    elif m == "dram__bytes_write.sum": d["wr"] = v * scale_b.get(u, 1.0)
agg = {}
for (kid, name), d in per.items():
    a = agg.setdefault(name, dict(n=0, us=0.0, rd=0.0, wr=0.0))
    a["n"] += 1; a["us"] += d.get("us", 0.0); a["rd"] += d.get("rd", 0.0); a["wr"] += d.get("wr", 0.0)
tot = sum(a["us"] for a in agg.values())
print(f"{'kernel':60s} {'launches':>8s} {'total ms':>9s} {'share':>6s} {'mean us':>8s} {'rd MB/l':>8s} {'wr MB/l':>8s} {'GB/s':>7s}")
for name, a in sorted(agg.items(), key=lambda kv: -kv[1]["us"]):
    gbs = (a["rd"] + a["wr"]) / (a["us"] * 1e-6) / 1e9 if a["us"] else 0
    print(f"{name[:60]:60s} {a['n']:8d} {a['us']/1e3:9.3f} {100*a['us']/tot:5.1f}% {a['us']/a['n']:8.1f} {a['rd']/a['n']/1e6:8.2f} {a['wr']/a['n']/1e6:8.2f} {gbs:7.0f}")
print(f"total {tot/1e3:.3f} ms over {sum(a['n'] for a in agg.values())} launches")
