"""Summarise an `ncu --csv` launch list (tools/ncu_raster_launches.sh): per kernel name, launches, mean device time,
share of the total, and the mean of the other collected metrics (issue% = warp instructions / duration / (132 SMs x 4
schedulers x 1980 MHz), computed here).  usage: python tools/summarize_launches.py FILE [skip_first_n] [--json OUT]
--json writes {kernel: {us, warp_inst, dram_bytes, ...}, "csrc_sha": <hash of the CUDA sources the capture was built
from>} -- the file bench.py reads `roofline.traffic` / `issue_frac` from (never a literal in bench.py)."""
import csv
import hashlib
import json
import sys
from pathlib import Path
from collections import OrderedDict, defaultdict

ISSUE_PEAK = 132 * 4 * 1.98e9      # warp instructions / s (H100 SXM)
argv = [a for a in sys.argv[1:]]
json_out = None
if "--json" in argv:
    i = argv.index("--json")
    json_out = argv[i + 1]
    del argv[i:i + 2]
path = argv[0]
skip = int(argv[1]) if len(argv) > 1 else 0


def csrc_sha() -> str:
    root = Path(__file__).resolve().parents[1] / "pixelsplat_b200" / "csrc"
    h = hashlib.sha1()
    for f in sorted(list(root.glob("*.cu")) + list(root.glob("*.cuh")) + [root / "Makefile"]):
        h.update(f.name.encode() + b"\0" + f.read_bytes())
    return h.hexdigest()[:16]


rows = []
with open(path) as f:
    lines = [l for l in f if not l.startswith("==")]
rd = csv.DictReader(lines)
per_id = OrderedDict()
for r in rd:
    k = r["ID"]
    per_id.setdefault(k, {"name": r["Kernel Name"], "grid": r.get("Grid Size", ""), "block": r.get("Block Size", "")})
    try:
        per_id[k][r["Metric Name"]] = float(r["Metric Value"].replace(",", ""))
    except ValueError:
        pass
launches = list(per_id.values())[skip:]
agg = defaultdict(lambda: defaultdict(float))
cnt = defaultdict(int)
for l in launches:
    n = l["name"].split("(")[0]
    cnt[n] += 1
    for k, v in l.items():
        if isinstance(v, float):
            agg[n][k] += v
total = sum(a["gpu__time_duration.sum"] for a in agg.values())
print(f"{len(launches)} launches, total {total/1e3:.1f} us")
print(f"{'kernel':44s} {'n':>4s} {'us':>8s} {'share':>6s} {'warps%':>7s} {'issue%':>7s} {'Minst':>8s} {'dramMB':>8s} {'regs':>5s}")
for n, a in sorted(agg.items(), key=lambda kv: -kv[1]["gpu__time_duration.sum"]):
    c = cnt[n]
    g = lambda k: a.get(k, 0.0) / c
    issue = g('smsp__inst_executed.sum') / max(g('gpu__time_duration.sum') * 1e-9, 1e-12) / ISSUE_PEAK * 100
    print(f"{n[:44]:44s} {c:4d} {g('gpu__time_duration.sum')/1e3:8.1f} {a['gpu__time_duration.sum']/total*100:5.1f}% "
          f"{g('sm__warps_active.avg.pct_of_peak_sustained_active'):7.1f} {issue:7.1f} "
          f"{g('smsp__inst_executed.sum')/1e6:8.2f} {(g('dram__bytes_read.sum')+g('dram__bytes_write.sum'))/1e6:8.2f} "
          f"{g('launch__registers_per_thread'):5.0f}")

if json_out:
    out = {"source": Path(path).name, "csrc_sha": csrc_sha(), "note": "per-launch means; ncu launch list (cold cache, serialised)"}
    import re
    for n, a in agg.items():
        c = cnt[n]
        if "ps::" not in n:
            continue
        key = re.sub(r"<.*>$", "", n.replace("void ", "").replace("ps::", "").strip())    # k_composite_bwd2<4> -> k_composite_bwd2
        out[key] = {
            "launches": c, "us": a["gpu__time_duration.sum"] / c / 1e3, "warp_inst": a.get("smsp__inst_executed.sum", 0.0) / c,
            "dram_bytes": (a.get("dram__bytes_read.sum", 0.0) + a.get("dram__bytes_write.sum", 0.0)) / c,
            "warps_active_pct": a.get("sm__warps_active.avg.pct_of_peak_sustained_active", 0.0) / c,
            "registers": a.get("launch__registers_per_thread", 0.0) / c}
    Path(json_out).write_text(json.dumps(out, indent=1))
    print("wrote", json_out)
