"""Summarise an `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv` launch list per kernel
family (the LAST of the captured steps): launches, time, share of the step, DRAM traffic, DRAM rate.
usage: python tools/ncu_launch_summary.py launches.csv [steps] > launches.md"""
import collections, csv, json, re, sys

path = sys.argv[1]
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
with open(path) as f:
    lines = [l for l in f if not l.startswith("==")]
per = collections.OrderedDict()
UNIT = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
for row in csv.DictReader(lines):
    d = per.setdefault(row["ID"], {"name": row["Kernel Name"], "grid": row["Grid Size"], "block": row["Block Size"]})
    v = float(row["Metric Value"].replace(",", ""))
    u, m = row["Metric Unit"], row["Metric Name"]
    if m == "gpu__time_duration.sum":
        d["us"] = v / 1000 if u.startswith("n") else (v if u.startswith("u") else v * 1000)
    elif m == "dram__bytes_read.sum":
        d["rd"] = v * UNIT[u]
    elif m == "dram__bytes_write.sum":
        d["wr"] = v * UNIT[u]

def short(name):
    m = re.search(r"(\w+_kernel\w*|\w+)\s*(<|\()", name.replace("void ", "").replace("(anonymous namespace)::", ""))
    return m.group(1) if m else name[:40]

ids = list(per)
ours = [i for i in ids if "at::" not in per[i]["name"]]
n_step = len(ours) // steps
last = ours[-n_step:]
fam = collections.OrderedDict()
for i in last:
    d = per[i]
    f = fam.setdefault(short(d["name"]), [0, 0.0, 0.0, 0.0])
    f[0] += 1; f[1] += d["us"]; f[2] += d.get("rd", 0); f[3] += d.get("wr", 0)
tot = sum(f[1] for f in fam.values())
print("| kernel | launches | time (us) | share | DRAM read (MB) | DRAM write (MB) | DRAM GB/s |")
print("|---|---|---|---|---|---|---|")
out = {}
for n, f in sorted(fam.items(), key=lambda x: -x[1][1]):
    print("| %s | %d | %.1f | %.1f%% | %.1f | %.1f | %.0f |" % (n, f[0], f[1], 100 * f[1] / tot, f[2] / 1e6, f[3] / 1e6, (f[2] + f[3]) / max(f[1], 1e-9) / 1e3))
    out[n] = dict(launches=f[0], us=round(f[1], 1), share=round(f[1] / tot, 4), dram_bytes=int(f[2] + f[3]), dram_bytes_per_launch=int((f[2] + f[3]) / f[0]))
print("\ntotal: %d launches, %.1f us (serialised, cold caches: shares, not absolutes, compare with the CUDA-event timing)" % (len(last), tot))
if len(sys.argv) > 3:
    json.dump(out, open(sys.argv[3], "w"), indent=1)
