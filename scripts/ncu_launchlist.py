"""Aggregate an `ncu --csv` launch list (gpu__time_duration.sum, dram bytes) per kernel name:
   python scripts/ncu_launchlist.py launches.csv > launches_summary.txt"""
import csv, sys, collections, re

def main(path):
    rows = []
    with open(path, newline="") as f:
        lines = [l for l in f if not l.startswith("==")]
    rd = csv.DictReader(lines)
    per = collections.defaultdict(lambda: collections.defaultdict(float))
    cnt = collections.Counter()
    seen = set()
    for r in rd:
        name = r.get("Kernel Name", "?")
        name = re.sub(r"\(.*", "", name)[:70]
        metric = r.get("Metric Name"); val = r.get("Metric Value", "0").replace(",", "")
        unit = r.get("Metric Unit", "")
        try: v = float(val)
        except ValueError: continue
        scale = {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3, "byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1.0)
        per[name][metric] += v * scale
        key = (r.get("ID"), name)
        if key not in seen:
            seen.add(key); cnt[name] += 1
    tot = sum(d.get("gpu__time_duration.sum", 0.0) for d in per.values())
    print(f"{'kernel':70s} {'launches':>8s} {'ms':>10s} {'share':>7s} {'dram MB/launch':>15s}")
    for name, d in sorted(per.items(), key=lambda kv: -kv[1].get("gpu__time_duration.sum", 0.0)):
        t = d.get("gpu__time_duration.sum", 0.0)
        by = d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)
        print(f"{name:70s} {cnt[name]:8d} {t:10.2f} {100*t/max(tot,1e-9):6.1f}% {by/max(cnt[name],1)/1e6:15.2f}")
    print(f"total kernel time under ncu: {tot:.1f} ms over {sum(cnt.values())} launches")

if __name__ == "__main__":
    main(sys.argv[1])
