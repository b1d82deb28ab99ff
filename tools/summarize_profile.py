"""Summarise the ncu outputs of tools/gpu_call_final2.sh into the tracked evidence files:
     python tools/summarize_profile.py gpurun_out/<dir> profiles/<tag> "<title>"
   <dir>/launches.csv.gz  (ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv of tools/profile_step.py 2)
        -> <tag>_launch_summary.md (per-kernel launches, time, share, DRAM bytes of ONE step) and <tag>_launches.csv.gz (copy)
        -> <tag>_traffic.json (DRAM bytes per launch of the level-0 kernels bench.py reports a roofline for)
   <dir>/full_raw.csv     (ncu --set full ... --page raw --csv), optional -> <tag>_ncu_full_summary.md"""
import collections
import csv
import gzip
import json
import os
import shutil
import sys


def read_launches(path):
    op = gzip.open if path.endswith(".gz") else open
    with op(path, "rt") as f:
        lines = [l for l in f if not l.startswith("==")]
    per = collections.OrderedDict()
    for r in csv.DictReader(lines):
        d = per.setdefault(int(r["ID"]), {"name": r["Kernel Name"], "grid": r["Grid Size"]})
        d[r["Metric Name"]] = (float(r["Metric Value"].replace(",", "")), r["Metric Unit"])
    out = []
    for i, d in per.items():
        def val(name, scale):
            v, u = d.get(name, (0.0, ""))
            return v * scale.get(u, 1.0)
        ns = val("gpu__time_duration.sum", {"ns": 1.0, "us": 1e3, "ms": 1e6, "nsecond": 1.0, "usecond": 1e3, "msecond": 1e6, "second": 1e9})
        byt = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
        out.append({"id": i, "name": d["name"], "ns": ns, "rd": val("dram__bytes_read.sum", byt), "wr": val("dram__bytes_write.sum", byt)})
    return out


def short(name):
    name = name.replace("void ", "").replace("dawn::(anonymous namespace)::", "dawn::").replace("dawn::<unnamed>::", "dawn::")
    return name.split("(")[0] if "<" not in name.split("(")[0] else name[:name.index(">(") + 1] if ">(" in name else name[:80]


def main(src, tag, title):
    launches = read_launches(os.path.join(src, "launches.csv.gz"))
    # one step = the launches after the last rotary_table/first-step marker: profile_step.py runs 2 steps; take the last 235 + torch tail
    n_step = 235
    names = [l["name"] for l in launches]
    tail = [i for i, n in enumerate(names) if n.startswith("void at::") or n.startswith("at::")]
    end = min(tail[-2:]) if len(tail) >= 2 else len(launches)
    step = launches[end - n_step:end]
    agg = collections.OrderedDict()
    for l in step:
        a = agg.setdefault(short(l["name"]), [0, 0.0, 0.0])
        a[0] += 1; a[1] += l["ns"]; a[2] += l["rd"] + l["wr"]
    tot_ns = sum(a[1] for a in agg.values()); tot_b = sum(a[2] for a in agg.values())
    rd = sum(l["rd"] for l in step); wr = sum(l["wr"] for l in step)
    with open(tag + "_launch_summary.md", "w") as f:
        f.write(f"# {title} — ncu launch list of one denoising step (H100, 200 f x 64x64, {len(step)} launches)\n\n")
        f.write("Command: `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none --csv python "
                "tools/profile_step.py 2` (`tools/gpu_call_final2.sh`; the last full step of the script; per-launch times are cold-cache / "
                "serialised: compare SHARES).  Summarised by `tools/summarize_profile.py`.\n\n")
        f.write(f"**Whole step: {tot_ns / 1e6:.2f} ms under ncu, DRAM traffic {rd / 1e9:.2f} GB read + {wr / 1e9:.2f} GB written = "
                f"{tot_b / 1e9:.2f} GB against B_alg = 22.9 GB (SURVEY 8d): {tot_b / 22.9e9:.2f}x.**\n\n")
        f.write("| kernel | launches | total ms | share | DRAM GB |\n|---|---:|---:|---:|---:|\n")
        for k, (n, ns, b) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| `{k[:70]}` | {n} | {ns / 1e6:.3f} | {100 * ns / tot_ns:.1f}% | {b / 1e9:.2f} |\n")
    shutil.copy(os.path.join(src, "launches.csv.gz"), tag + "_launches.csv.gz")

    def per_launch(pred, pick_max=True):
        xs = [l for l in step if pred(l["name"])]
        if not xs:
            return None
        if pick_max:                      # the level-0 launches are the largest of their kind
            mx = max(l["rd"] + l["wr"] for l in xs)
            xs = [l for l in xs if l["rd"] + l["wr"] > 0.8 * mx]
        return {"dram_bytes_per_launch": sum(l["rd"] + l["wr"] for l in xs) / len(xs), "launches_captured": len(xs),
                "ncu_ms": sum(l["ns"] for l in xs) / len(xs) / 1e6}
    traffic = {"source": f"ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum --clock-control none, {title} "
                         f"({os.path.basename(tag)}_launch_summary.md): bytes per launch at the bench shape (200 f x 64x64), level-0 launches of one step",
               "temporal_fused_l0": per_launch(lambda n: "temporal_fused_kernel" in n),
               "conv3x3_l0": per_launch(lambda n: "tc_conv3_kernel<64" in n, pick_max=False),      # every 64-output-channel (= level-0) 3x3 conv of the step
               "gn_apply_l0": per_launch(lambda n: "gn_apply_kernel" in n),
               "whole_step": {"dram_bytes": tot_b, "ncu_ms": tot_ns / 1e6, "launches": len(step)}}
    raw = os.path.join(src, "full_raw.csv")
    if os.path.exists(raw):
        # where the --set full capture holds the kernel, its DRAM bytes replace the metrics-pass ones (the roofline contract names --set full)
        rows = list(csv.reader(open(raw)))
        hdr, units, data = rows[0], rows[1], rows[2:]
        byt = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
        tms = {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}
        cr = [i for i, h in enumerate(hdr) if h.endswith("dram__bytes_read.sum")][0]
        cw = [i for i, h in enumerate(hdr) if h.endswith("dram__bytes_write.sum")][0]
        cd = [i for i, h in enumerate(hdr) if h.endswith("gpu__time_duration.sum")][0]
        for cat, pat in (("temporal_fused_l0", "temporal_fused_kernel"), ("conv3x3_l0", "tc_conv3_kernel<64"), ("gn_apply_l0", "gn_apply_kernel")):
            xs = [r for r in data if pat in r[4]]
            if xs:
                traffic[cat] = {"dram_bytes_per_launch": sum(float(r[cr]) * byt[units[cr]] + float(r[cw]) * byt[units[cw]] for r in xs) / len(xs),
                                "launches_captured": len(xs), "ncu_ms": sum(float(r[cd]) * tms[units[cd]] for r in xs) / len(xs),
                                "source": "ncu --set full (" + os.path.basename(tag) + "_ncu_full_summary.md)"}
    with open(tag + "_traffic.json", "w") as f:
        json.dump(traffic, f, indent=1)
    print(open(tag + "_launch_summary.md").read()[:3000])
    print(json.dumps(traffic, indent=1))

    raw = os.path.join(src, "full_raw.csv")
    if os.path.exists(raw):
        rows = list(csv.reader(open(raw)))
        hdr, units, data = rows[0], rows[1], rows[2:]
        want = [("duration", "gpu__time_duration.sum"), ("DRAM read", "dram__bytes_read.sum"), ("DRAM write", "dram__bytes_write.sum"),
                ("tensor pipe active %", "sm__inst_executed_pipe_tensor_op_hmma.avg.pct_of_peak_sustained_active"),
                ("tensor pipe (any) active %", "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active"),
                ("achieved occupancy %", "sm__warps_active.avg.pct_of_peak_sustained_active"), ("registers/thread", "launch__registers_per_thread"),
                ("dynamic smem/block", "launch__shared_mem_per_block_dynamic"), ("issue slots busy %", "sm__inst_issued.avg.pct_of_peak_sustained_active"),
                ("L2 hit rate %", "lts__t_sector_hit_rate.pct"),
                ("stall long_scoreboard", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio"),
                ("stall barrier", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio"),
                ("stall wait", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio"),
                ("stall short_scoreboard", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio")]
        with open(tag + "_ncu_full_summary.md", "w") as f:
            f.write(f"# {title} — `ncu --set full --clock-control none --import-source on`, {len(data)} launches (H100, 200 f x 64x64; `tools/gpu_call_ncufull.sh`)\n\n")
            f.write("| metric | " + " | ".join(f"launch {i}" for i in range(len(data))) + " |\n|---|" + "---:|" * len(data) + "\n")
            f.write("| kernel | " + " | ".join(short(r[4])[:44] for r in data) + " |\n")
            for label, key in want:
                c = [i for i, h in enumerate(hdr) if h.endswith(key)]
                if not c:
                    continue
                f.write(f"| {label} ({units[c[0]]}) | " + " | ".join(r[c[0]] for r in data) + " |\n")
        print(open(tag + "_ncu_full_summary.md").read()[:2500])


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3])
