"""`ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv` launch list of one optimizer step
(tools/one_step.py) -> per-kernel table (launches, total us, DRAM MB, GB/s) and the DRAM bytes per launch of the tensor-core
convolutions.
usage: launch_traffic.py launches.csv [out.json]"""
import collections
import csv
import json
import sys

rows = list(csv.reader(open(sys.argv[1])))
hdr = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
H = rows[hdr]
ki, ii, mi, vi, ui = H.index("Kernel Name"), H.index("ID"), H.index("Metric Name"), H.index("Metric Value"), H.index("Metric Unit")
per = collections.OrderedDict()
for r in rows[hdr + 1:]:
    e = per.setdefault(r[ii], {'name': r[ki]})
    v = float(r[vi].replace(",", ""))
    u = r[ui]
    if r[mi].startswith('gpu__time'):
        e['us'] = v / 1e3 if u in ('ns', 'nsecond') else (v * 1e3 if u in ('ms', 'msecond') else v)
    else:
        scale = {'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9}.get(u, 1.0)
        e[r[mi]] = v * scale
agg = collections.defaultdict(lambda: [0, 0.0, 0.0])
for e in per.values():
    k = e['name'].split("(")[0].replace("void ", "").replace("<unnamed>::", "")[:58]
    a = agg[k]
    a[0] += 1; a[1] += e.get('us', 0.0); a[2] += e.get('dram__bytes_read.sum', 0.0) + e.get('dram__bytes_write.sum', 0.0)
tot = sum(a[1] for a in agg.values())
print("launches: %d   sum of durations %.1f us (serialised, cold caches: shares matter, not absolutes)" % (len(per), tot))
print("%10s %6s %5s %10s %9s  %s" % ("us", "share", "n", "DRAM MB", "GB/s", "kernel"))
for k, (c, us, by) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:40]:
    print("%10.1f %5.1f%% %5d %10.1f %9.0f  %s" % (us, 100 * us / tot, c, by / 1e6, by / us / 1e3 if us else 0, k))
conv = [(c, us, by) for k, (c, us, by) in agg.items() if k.startswith('conv_tc')]
n = sum(c for c, _, _ in conv)
if n and len(sys.argv) > 2:
    out = {"source": "%s (ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum of tools/one_step.py)" % sys.argv[1],
           "kernels": "conv_tc_kernel<*> + conv_tc2_kernel<*> + conv_tc4_kernel<*> (fwd + dgrad launches of one optimizer step, config 3)",
           "launches": n, "dram_bytes_per_launch": sum(by for _, _, by in conv) / n,
           "avg_us_per_launch_under_ncu": sum(us for _, us, _ in conv) / n,
           "share_of_step_under_ncu": sum(us for _, us, _ in conv) / tot}
    json.dump(out, open(sys.argv[2], 'w'), indent=1)
    print(json.dumps(out))
