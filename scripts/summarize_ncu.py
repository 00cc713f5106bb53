"""Summarise ncu captures (runs/<tag>/) into a markdown file <name>.md."""
import csv, json, subprocess, sys, os, collections

tag, out = sys.argv[1], sys.argv[2]
d = f"runs/{tag}"
L = []
L.append(f"# ncu summary `{tag}` (H100, sm_90a)\n")
L.append("Source: `scripts/gpu_final_r2.sh` (round 1: `scripts/gpu_round.sh`) -> `ncu --set full --clock-control none --import-source on` on "
         "`python bench.py --profile --steps 8 --warmup 3` (1M groups x 5 peers, 4 arenas rotated), and the "
         "`--metrics gpu__time_duration.sum` launch list of the same command.  ncu serialises kernels and "
         "replays them, so absolute times are cold-cache; compare SHARES with the live CUDA-event numbers "
         "in bench.py.\n")
def launch_table(path, title):
    if not os.path.exists(path):
        return
    rows = list(csv.reader(open(path, errors="ignore")))
    hdr, per = None, collections.defaultdict(list)
    for r in rows:
        if "Kernel Name" in r:
            hdr = r
            continue
        if hdr and len(r) == len(hdr):
            x = dict(zip(hdr, r))
            if x.get("Metric Name") == "gpu__time_duration.sum":
                v = float(x["Metric Value"].replace(",", ""))
                per[x["Kernel Name"].split("(")[0]].append(v / 1e3 if x["Metric Unit"] == "ns" else v)
    tot = sum(sum(v) for v in per.values())
    L.append(f"## {title}\n\n| kernel | launches | avg us | min | max | share |\n|---|---|---|---|---|---|")
    for k, v in sorted(per.items(), key=lambda kv: -sum(kv[1])):
        L.append(f"| `{k}` | {len(v)} | {sum(v)/len(v):.2f} | {min(v):.2f} | {max(v):.2f} | {sum(v)/tot:.1%} |")
    L.append("")

launch_table(f"{d}/launches.csv", "Launch list, default path (gpu__time_duration.sum)")
launch_table(f"{d}/launches_scatter.csv", "Launch list, `--scatter` path (gpu__time_duration.sum)")
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__warps_eligible.avg.per_cycle_active",
        "smsp__inst_executed.sum", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
        "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
        "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum"]
for name in ("fused", "fused_cfg4", "compact", "ctile", "recompute", "apply", "wire"):
    rep = f"{d}/prof_{name}.ncu-rep"
    if not os.path.exists(rep):
        continue
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    for row in rows[2:]:
        x = dict(zip(hdr, row))
        L.append(f"\n## `{x['Kernel Name'][:70]}` (`prof_{name}`, ncu --set full, launch id {x['ID']})\n\n| metric | value | unit |\n|---|---|---|")
        for w in want:
            if w in x:
                L.append(f"| {w} | {x[w]} | {units[hdr.index(w)]} |")
        st = sorted(((k, float(v.replace(',', '') or 0)) for k, v in x.items()
                     if "average_warps_issue_stalled" in k and k.endswith("_per_issue_active.ratio")), key=lambda kv: -kv[1])
        L.append("\nTop warp stall reasons (warps stalled per issue-active cycle): " +
                 ", ".join(f"{k.split('issue_stalled_')[1].replace('_per_issue_active.ratio','')} {v:.2f}" for k, v in st[:5]))
        rd, wr = float(x["dram__bytes_read.sum"].replace(",", "")), float(x["dram__bytes_write.sum"].replace(",", ""))
        ur, uw = units[hdr.index("dram__bytes_read.sum")], units[hdr.index("dram__bytes_write.sum")]
        L.append(f"\nDRAM traffic per launch: read {rd} {ur} + write {wr} {uw}.")
for extra, title in (("sass_summary.txt", "SASS mnemonics (cuobjdump -sass of the shipped libraftgpu.so): 1-D bulk TMA (UBLKCP), mbarrier (SYNCS), warp reductions (REDUX)"),
                     ("micro_tile.txt", "scripts/micro_tile.py on the same box (CUDA events; phase switches are diagnostics)")):
    if os.path.exists(f"{d}/{extra}"):
        L.append(f"\n## {title}\n\n```\n" + open(f"{d}/{extra}").read().rstrip() + "\n```")
for w_ in ("cfg3", "cfg4", "cfg5", "reference"):
    if os.path.exists(f"{d}/bench_{w_}.json"):
        try:
            bj = json.loads(open(f"{d}/bench_{w_}.json").read().strip().splitlines()[-1])
            L.append(f"\n## bench.py {'--impl reference' if w_ == 'reference' else '--workload ' + w_} --steps 20 --warmup 5 (live, not under ncu)\n\n```json\n" + json.dumps(bj, indent=1) + "\n```")
        except Exception as e:
            L.append(f"\n(bench_{w_}.json unreadable: {e})")
try:
    b = json.loads(open(f"{d}/bench.json").read().strip().splitlines()[-1])
    L.append("\n## bench.py line of the same build (live CUDA events, not under ncu)\n\n```json\n" + json.dumps(b, indent=1) + "\n```")
    if os.path.exists(f"{d}/bench_compact.json"):
        b3 = json.loads(open(f"{d}/bench_compact.json").read().strip().splitlines()[-1])
        L.append("\n## bench.py --compact-device (compact stream + its fused kernel, device-resident leg) of the same build\n\n```json\n" + json.dumps(b3, indent=1) + "\n```")
    if os.path.exists(f"{d}/bench_scatter.json"):
        b2 = json.loads(open(f"{d}/bench_scatter.json").read().strip().splitlines()[-1])
        L.append("\n## bench.py --scatter (general two-kernel path) of the same build\n\n```json\n" + json.dumps(b2, indent=1) + "\n```")
except Exception as e:
    L.append(f"\n(no bench.json: {e})")
open(out, "w").write("\n".join(L) + "\n")
print("wrote", out)
