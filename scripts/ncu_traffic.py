"""DRAM bytes per launch of the dominant kernel family from an ncu launch-list summary (scripts/ncu_launchlist.py):
    python scripts/ncu_traffic.py <summary.txt> <n_gpus> <out.json>
merges {"<n_gpus>": {"gemm_wgmma_kernel": {...}}} into the JSON bench.py reads for roofline.traffic."""
import json
import re
import sys
from pathlib import Path


def main(summary, n_gpus, out):
    tot_bytes = tot_launch = tot_ms = all_ms = 0.0
    for line in Path(summary).read_text().splitlines():
        m = re.match(r"(.+?)\s+(\d+)\s+([\d.]+)\s+([\d.]+)%\s+([\d.]+)\s*$", line)
        if not m:
            continue
        name, cnt, ms, mb = m.group(1), int(m.group(2)), float(m.group(3)), float(m.group(5))
        all_ms += ms
        if "gemm_wgmma_kernel" in name:
            tot_bytes += cnt * mb * 1e6
            tot_launch += cnt
            tot_ms += ms
    p = Path(out)
    d = json.loads(p.read_text()) if p.exists() else {}
    d = {k: v for k, v in d.items() if k.isdigit()}
    d[str(n_gpus)] = {"gemm_wgmma_kernel": {
        "dram_bytes_per_launch": round(tot_bytes / max(tot_launch, 1)),
        "source": f"{Path(summary).name}: sum over the gemm_wgmma_kernel instantiations of launches x (dram__bytes_read.sum "
                  f"+ dram__bytes_write.sum) / {int(tot_launch)} launches of one clip (ncu launch list of bench.py --one-clip)",
        "share_of_step_under_ncu": round(tot_ms / max(all_ms, 1e-9), 4)}}
    p.write_text(json.dumps(d, indent=1))
    print(json.dumps(d[str(n_gpus)]))


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]), sys.argv[3])
