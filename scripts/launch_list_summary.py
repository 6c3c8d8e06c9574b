"""Per-kernel launch count / mean duration / share of an `ncu --metrics gpu__time_duration.sum --csv` log:
python scripts/launch_list_summary.py <launches.csv> > <name>.txt"""
import collections, csv, sys
rows = [r for r in csv.reader(l for l in open(sys.argv[1]) if l.startswith('"'))]
hdr = rows[0]; ik, iv, iu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
tot = collections.defaultdict(float); cnt = collections.Counter()
for r in rows[1:]:
    v = float(r[iv].replace(",", "")); u = r[iu]
    ms = v / 1e6 if u in ("ns", "nsecond") else (v / 1e3 if u in ("us", "usecond") else (v if u in ("ms", "msecond") else v * 1e3))
    k = r[ik].split("(")[0].replace("void ", "").replace("b200::", "")
    tot[k] += ms; cnt[k] += 1
s = sum(tot.values())
print(f"{'kernel':62s} launches   mean ms   share")
for k, v in sorted(tot.items(), key=lambda x: -x[1]):
    print(f"{k:62s} {cnt[k]:8d} {v / cnt[k]:9.3f} {100 * v / s:6.1f} %")
